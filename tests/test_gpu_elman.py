"""The Elman RNN on the GPU: ``RNN`` (the Elman instantiations of csrc/rnn_anyh.cu) and ``RNNCell`` (cell.cu),
nonlinearity tanh and relu.

Reference: stock torch.nn.RNN / RNNCell in float64 on CPU. Tolerances as tests/test_gpu_any_hidden.py: outputs and
states 1e-5 (absolute for tanh; relative to the largest entry for relu, whose outputs are unbounded), gradients 1e-4
relative to the largest entry of each tensor (dx, dh_0, every dW and db). The per-step test holds each step of the
kernel's own trajectory to kappa * u * S away from default init (tests/test_gpu_numerics_f64.py). Which config each
shape runs is read from the B200RNN_DEBUG lines of a subprocess: every Elman instantiation and both weight tiers are
reached."""
import contextlib
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

import b200rnn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OUT_TOL = 1e-5
GRAD_RTOL = 1e-4
TF32_GRAD_RTOL = 4e-3   # single-pass TF32 operands (tests/test_gpu_cells.py)
KAPPA = 24.0
U32, U_TF32 = 2.0 ** -24, 2.0 ** -11
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONLIN = ("tanh", "relu")


def _np(t):
    return t.detach().cpu().double().numpy()


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max(initial=0.0) / max(np.abs(b).max(initial=0.0), 1e-30))


def _out_err(nl, a, b):
    """absolute for tanh (|h| <= 1), relative to the largest entry for relu"""
    d = float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max(initial=0.0))
    return d if nl == "tanh" else d / max(float(np.abs(np.asarray(b)).max(initial=0.0)), 1.0)


@contextlib.contextmanager
def _tf32(on):
    old = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32" if on else "ieee"
    try:
        yield
    finally:
        torch.backends.cuda.matmul.fp32_precision = old


def _compare(nl, ref, mine, x, *, bf=False, lens=None, h0=None, h0_grad=False, seed=11):
    """Forward and backward of ``mine`` (GPU) against ``ref`` in float64 on CPU, same inputs and output weights:
    y, h_n, dx, dh_0 and every parameter gradient"""
    g = torch.Generator().manual_seed(seed)
    ref64 = ref.double()
    T = x.shape[1] if bf else x.shape[0]

    def run(model, dev, dtype):
        model.zero_grad(set_to_none=True)
        xx = x.to(dev, dtype).requires_grad_(True)
        hh = h0.to(dev, dtype).requires_grad_(h0_grad) if h0 is not None else None
        inp = pack_padded_sequence(xx, lens, batch_first=bf, enforce_sorted=False) if lens is not None else xx
        y, hn = model(inp, hh)
        if lens is not None:
            y = pad_packed_sequence(y, batch_first=bf, total_length=T)[0]
        return xx, hh, y, hn

    xm, hm, ym, hnm = run(mine, DEV, torch.float32)
    xr, hr, yr, hnr = run(ref64, "cpu", torch.float64)
    wy = torch.randn(yr.shape, generator=g, dtype=torch.float64)
    wh = torch.randn(hnr.shape, generator=g, dtype=torch.float64)
    ((ym * wy.to(DEV, torch.float32)).sum() + (hnm * wh.to(DEV, torch.float32)).sum()).backward()
    ((yr * wy).sum() + (hnr * wh).sum()).backward()
    torch.cuda.synchronize()
    assert _out_err(nl, _np(ym), _np(yr)) <= OUT_TOL
    assert _out_err(nl, _np(hnm), _np(hnr)) <= OUT_TOL
    assert _rel(_np(xm.grad), _np(xr.grad)) <= GRAD_RTOL
    if h0_grad:
        assert _rel(_np(hm.grad), _np(hr.grad)) <= GRAD_RTOL
    elif hm is not None:
        assert hm.grad is None
    for (n, pr), pm in zip(ref64.named_parameters(), mine.parameters()):
        assert _rel(_np(pm.grad), _np(pr.grad)) <= GRAD_RTOL, n


@pytest.mark.parametrize("H", list(range(16, 1025, 16)))
def test_every_multiple_of_16_forward_and_backward(H):
    """Every accepted hidden size, tanh and relu, bidirectional, with hx and dh_0. Sizes whose H / 8 groups do not
    split evenly over the cluster give the CTAs unequal slices"""
    T, B, I = 5, 3, 24
    for nl in NONLIN:
        torch.manual_seed(H)
        ref = torch.nn.RNN(I, H, nonlinearity=nl, bidirectional=True)
        mine = b200rnn.from_torch(ref).to(DEV)
        g = torch.Generator().manual_seed(H + 1)
        x = torch.randn(T, B, I, generator=g)
        h0 = 0.5 * torch.randn(2, B, H, generator=g)
        _compare(nl, ref, mine, x, h0=h0, h0_grad=True)


# nonlinearity, H, I, L, bidirectional, batch_first, B, T
MATRIX = [
    ("tanh", 64, 40, 1, False, False, 1, 1),
    ("relu", 64, 40, 1, False, True, 16, 7),
    ("tanh", 128, 64, 2, True, False, 64, 7),
    ("relu", 128, 33, 3, False, True, 200, 7),
    ("tanh", 256, 128, 1, False, False, 128, 120),
    ("relu", 256, 64, 2, True, True, 3, 120),
    ("tanh", 96, 13, 3, True, True, 200, 1),
    ("relu", 512, 64, 1, True, False, 64, 7),
    ("tanh", 512, 48, 2, False, False, 3, 120),
    ("relu", 1024, 100, 1, False, True, 16, 7),
    ("tanh", 1024, 64, 2, True, False, 200, 7),
    ("relu", 48, 30, 2, True, False, 128, 120),
]


@pytest.mark.parametrize("nl, H, I, L, bi, bf, B, T", MATRIX,
                         ids=[f"{c[0]}{c[1]}_I{c[2]}_L{c[3]}_D{2 if c[4] else 1}_{'bf' if c[5] else 'tm'}_B{c[6]}_T{c[7]}"
                              for c in MATRIX])
def test_matrix_against_float64(nl, H, I, L, bi, bf, B, T):
    torch.manual_seed(H + L + T)
    ref = torch.nn.RNN(I, H, num_layers=L, nonlinearity=nl, bidirectional=bi, batch_first=bf)
    mine = b200rnn.from_torch(ref).to(DEV)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(*((B, T, I) if bf else (T, B, I)), generator=g)
    _compare(nl, ref, mine, x, bf=bf)
    h0 = 0.5 * torch.randn(L * (2 if bi else 1), B, H, generator=g)
    _compare(nl, ref, mine, x, bf=bf, h0=h0, h0_grad=True)


@pytest.mark.parametrize("nl, H, B, scale", [("tanh", 64, 16, 3.0), ("tanh", 384, 5, 3.0), ("tanh", 1024, 3, 3.0),
                                             ("relu", 96, 16, 1.0), ("relu", 1024, 3, 1.0)])
def test_per_step_bound_at_t120_non_default_init(nl, H, B, scale):
    """Each step of a T = 120 launch, recomputed in float64 from the kernel's own h_{t-1} (its previous output), within
    KAPPA * u * (S + 1): S is the magnitude sum of the pre-activation's terms, the 1 covers the activation's own
    rounding. tanh: weights at 3x the default range and inputs x4, so that it saturates; relu: inputs x4"""
    T, I = 120, 40
    torch.manual_seed(H)
    m = b200rnn.RNN(I, H, nonlinearity=nl).to(DEV)
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(scale)
    x = 4.0 * torch.randn(T, B, I, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        y = _np(m(x.to(DEV))[0])
    w_ih, w_hh, b_ih, b_hh = [_np(p) for p in m.parameters()]
    xs = x.double().numpy()
    worst, h = 0.0, np.zeros((B, H))
    for t in range(T):
        pre = xs[t] @ w_ih.T + b_ih + b_hh + h @ w_hh.T
        S = np.abs(xs[t]) @ np.abs(w_ih).T + np.abs(b_ih) + np.abs(b_hh) + np.abs(h) @ np.abs(w_hh).T
        want = np.tanh(pre) if nl == "tanh" else np.maximum(pre, 0.0)
        worst = max(worst, float((np.abs(y[t] - want) / (KAPPA * U32 * (S + 1.0))).max()))
        h = y[t]
    print(f"RNN_{nl.upper()}-{H}: worst per-step err / bound = {worst:.3f}")
    assert worst <= 1.0


def _lengths(B, T, seed=5):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, T + 1, (B,), generator=g)
    lens[: B // 4] = torch.randint(1, 4, (B // 4,), generator=g)  # skewed: a quarter of very short rows
    lens[B // 2] = T
    return lens


@pytest.mark.parametrize("nl, H, B, T, bi, hx, hx_grad", [
    ("tanh", 96, 64, 40, False, False, False),
    ("relu", 48, 37, 30, True, True, True),
    ("tanh", 512, 20, 25, True, True, False),     # shared-memory tier, ragged, reverse direction
    ("relu", 1024, 19, 20, False, True, True),    # L2 tier, ragged
    ("tanh", 464, 13, 9, True, True, True),       # uneven slices: CTAs of 24 and 32 units
    ("relu", 1008, 6, 8, False, True, False),
])
def test_packed_sequence_and_hx(nl, H, B, T, bi, hx, hx_grad):
    """PackedSequence with skewed lengths, with and without an initial state, with and without dh_0"""
    I, L = 24, 2
    torch.manual_seed(3)
    ref = torch.nn.RNN(I, H, num_layers=L, nonlinearity=nl, bidirectional=bi, batch_first=True)
    mine = b200rnn.from_torch(ref).to(DEV)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(B, T, I, generator=g)
    h0 = 0.5 * torch.randn(L * (2 if bi else 1), B, H, generator=g) if hx else None
    _compare(nl, ref, mine, x, bf=True, lens=_lengths(B, T), h0=h0, h0_grad=hx_grad)


@pytest.mark.parametrize("nl, H", [("tanh", 128), ("relu", 320)])
def test_chunked_runs_are_bitwise_one_call(nl, H):
    """h_n of one chunk as hx of the next: the same outputs and final state, bit for bit, as one call over all steps"""
    T, B, I, L = 40, 24, 32, 2
    torch.manual_seed(2)
    m = b200rnn.RNN(I, H, num_layers=L, nonlinearity=nl, bidirectional=False).to(DEV)
    x = torch.randn(T, B, I, generator=torch.Generator().manual_seed(5)).to(DEV)
    h0 = 0.5 * torch.randn(L, B, H, generator=torch.Generator().manual_seed(6)).to(DEV)
    with torch.no_grad():
        y_all, hn_all = m(x, h0)
        h, ys = h0, []
        for t0 in range(0, T, 10):
            y, h = m(x[t0:t0 + 10], h)
            ys.append(y)
    assert torch.equal(torch.cat(ys), y_all) and torch.equal(h, hn_all)


@pytest.mark.parametrize("nl, H", [("tanh", 64), ("relu", 320)])
def test_unbatched_input(nl, H):
    torch.manual_seed(8)
    ref = torch.nn.RNN(20, H, num_layers=2, nonlinearity=nl, bidirectional=True)
    mine = b200rnn.from_torch(ref).to(DEV)
    ref64 = ref.double()
    x = torch.randn(9, 20)
    h0 = 0.5 * torch.randn(4, H)
    xm, xr = x.to(DEV).requires_grad_(True), x.double().requires_grad_(True)
    ym, yr = mine(xm, h0.to(DEV)), ref64(xr, h0.double())
    assert ym[0].shape == yr[0].shape and ym[1].shape == yr[1].shape
    assert _out_err(nl, _np(ym[0]), _np(yr[0])) <= OUT_TOL
    assert _out_err(nl, _np(ym[1]), _np(yr[1])) <= OUT_TOL
    ym[0].sum().backward()
    yr[0].sum().backward()
    assert _rel(_np(xm.grad), _np(xr.grad)) <= GRAD_RTOL


@pytest.mark.parametrize("nl, H", [("tanh", 64), ("relu", 128)])
def test_dropout_masks_of_forward_and_backward_agree(nl, H):
    """Train mode, p = 0.5, one step of one sequence: the units whose dW_ih_l1 column is zero are the ones the dropout
    zeroed; stock layer 1 on h0 * mask / (1 - p) reproduces the output (forward mask) and dx (backward mask)"""
    p = 0.5
    torch.manual_seed(6)
    m = b200rnn.RNN(32, H, num_layers=2, nonlinearity=nl, dropout=p, bidirectional=True).to(DEV).train()
    layers = [torch.nn.RNN(32 if i == 0 else 2 * H, H, nonlinearity=nl, bidirectional=True).double()
              for i in range(2)]
    with torch.no_grad():
        for i, mod in enumerate(layers):
            for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                for sfx in ("", "_reverse"):
                    getattr(mod, f"{n}_l0{sfx}").copy_(getattr(m, f"{n}_l{i}{sfx}").cpu())
    x = torch.randn(1, 1, 32)
    dy = torch.randn(1, 1, 2 * H)
    xm = x.to(DEV).requires_grad_(True)
    y, _ = m(xm)
    (y * dy.to(DEV)).sum().backward()
    kept = (m.weight_ih_l1.grad.abs().sum(0) != 0).cpu()
    frac = 1.0 - kept.double().mean().item()
    assert 0.2 < frac < 0.8, frac
    xr = x.double().requires_grad_(True)
    h0 = layers[0](xr)[0]
    y_check = layers[1](h0 * kept / (1 - p))[0]
    (y_check * dy.double()).sum().backward()
    assert _out_err(nl, _np(y), _np(y_check)) <= OUT_TOL
    assert _rel(_np(xm.grad), _np(xr.grad)) <= GRAD_RTOL


@pytest.mark.parametrize("nl, H, B", [("tanh", 384, 24), ("relu", 1024, 8)])
def test_tf32_mode_meets_the_emulation_bounds(nl, H, B):
    """torch's "tf32" matmul precision: the input projection and the gradient GEMMs go single-pass TF32 (I = 256 and H
    multiples of 128 put every GEMM on the tensor cores); the recurrence stays fp32. The float64 emulation below rounds
    exactly those operands with oracle/tf32.py's rounding, teacher-forced from the kernel's own outputs as Tf32RNN is"""
    from oracle.tf32 import round_tf32 as R

    T, I = 30, 256
    torch.manual_seed(0)
    m = b200rnn.RNN(I, H, nonlinearity=nl).to(DEV)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(T, B, I, generator=g)
    xm = x.to(DEV).requires_grad_(True)
    with _tf32(True):
        assert m._config().tf32
        y, hn = m(xm)
    dy = torch.randn(T, B, H, generator=g)
    dh = torch.randn(1, B, H, generator=g)
    ((y * dy.to(DEV)).sum() + (hn * dh.to(DEV)).sum()).backward()
    torch.cuda.synchronize()
    w_ih, w_hh, b_ih, b_hh = [_np(p) for p in m.parameters()]
    act = np.tanh if nl == "tanh" else (lambda a: np.maximum(a, 0.0))
    xs, ys = x.double().numpy(), _np(y)
    r = lambda a: R(a).astype(np.float64)  # noqa: E731
    gi = np.einsum("tbi,hi->tbh", r(xs), r(w_ih)) + b_ih + b_hh
    hp = np.concatenate([np.zeros((1, B, H)), ys[:-1]])          # the kernel's own h_{t-1}
    want = act(gi + hp @ w_hh.T)
    assert _out_err(nl, ys, want) <= OUT_TOL
    assert _out_err(nl, _np(hn)[0], want[-1]) <= OUT_TOL
    dyn, dhc = dy.double().numpy(), dh.double().numpy()[0]
    dpre = np.zeros((T, B, H))
    for t in range(T - 1, -1, -1):
        d = dyn[t] + dhc
        dpre[t] = d * (1.0 - ys[t] ** 2) if nl == "tanh" else d * (ys[t] > 0)  # from the saved h_t, as the kernel
        dhc = dpre[t] @ w_hh
    dx = np.einsum("tbh,hi->tbi", r(dpre), r(w_ih))
    dw_ih = np.einsum("tbh,tbi->hi", r(dpre), r(xs))
    dw_hh = np.einsum("tbh,tbk->hk", r(dpre[1:]), r(ys[:-1]))
    db = dpre.sum((0, 1))
    assert _rel(_np(xm.grad), dx) <= TF32_GRAD_RTOL
    for (n, p), want_g in zip(m.named_parameters(), (dw_ih, dw_hh, db, db)):
        assert _rel(_np(p.grad), want_g) <= TF32_GRAD_RTOL, n


@pytest.mark.parametrize("nl, H, B, bi", [("tanh", 96, 40, True), ("relu", 1024, 12, False)])
def test_repeatable_and_cuda_graph_replay_is_bitwise_eager(nl, H, B, bi):
    T, I = 20, 48
    torch.manual_seed(9)
    mine = b200rnn.RNN(I, H, num_layers=2, nonlinearity=nl, bidirectional=bi).to(DEV)
    D = 2 if bi else 1
    g = torch.Generator().manual_seed(3)
    x = torch.randn(T, B, I, generator=g).to(DEV)
    h0 = (0.5 * torch.randn(2 * D, B, H, generator=g)).to(DEV).requires_grad_(True)
    wy = torch.randn(T, B, D * H, generator=g).to(DEV)

    def step():
        y, hn = mine(x, h0)
        ((y * wy).sum() + hn.sum()).backward()
        return y.detach(), hn.detach()

    def clear():
        mine.zero_grad(set_to_none=True)
        h0.grad = None

    clear()
    eager = [*(t.clone() for t in step()), h0.grad.clone()] + [p.grad.clone() for p in mine.parameters()]
    clear()
    again = [*(t.clone() for t in step()), h0.grad.clone()] + [p.grad.clone() for p in mine.parameters()]
    for a, b in zip(again, eager):
        assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            clear()
            step()
    torch.cuda.current_stream().wait_stream(s)
    clear()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_g, hn_g = step()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    got = [y_g, hn_g, h0.grad] + [p.grad for p in mine.parameters()]
    for a, b in zip(got, eager):
        assert torch.equal(a, b)


_DISPATCH = r"""
import sys, torch, b200rnn
from torch.nn.utils.rnn import pack_padded_sequence
for nl, H, B in [("tanh", 512, 64), ("relu", 1024, 8), ("relu", 128, 200), ("tanh", 256, 16)]:
    for ragged in (False, True):
        torch.manual_seed(0)
        m = b200rnn.RNN(16, H, nonlinearity=nl).cuda()
        x = torch.randn(5, B, 16, device="cuda", requires_grad=True)
        print("SHAPE", nl, H, B, int(ragged), file=sys.stderr, flush=True)
        if ragged:
            lens = torch.arange(B) % 5 + 1
            y = m(pack_padded_sequence(x, lens, enforce_sorted=False))[0].data
        else:
            y = m(x)[0]
        y.sum().backward()
        torch.cuda.synchronize()
"""


def test_dispatch_reaches_every_instantiation_and_both_tiers():
    env = dict(os.environ, B200RNN_DEBUG="1")
    r = subprocess.run([sys.executable, "-c", _DISPATCH], capture_output=True, text=True, env=env,
                       cwd=os.path.join(ROOT, "icassp2022-depression_b200"), timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    pat = re.compile(r"\[b200rnn\] (fwd|bwd) elman cfg (RNN_TANH|RNN_RELU) VL=(\d) H=(\d+) C=(\d+) BS=(\d+) "
                     r"tier=(smem|l2): need (\d+) clusters, capacity (\d+), smem (\d+)")
    seen, modes = set(), set()
    for ln in r.stderr.splitlines():
        assert " anyh cfg RNN" not in ln and not re.search(r"\] (fwd|bwd) cfg ", ln), ln  # no fixed config, no anyh
        mt = pat.search(ln)
        if not mt:
            continue
        pas, mode, vl, H, C, BS, tier, need, cap, smem = mt.groups()
        H, C, BS, cap, smem = map(int, (H, C, BS, cap, smem))
        assert C in (2, 4, 8, 16) and C <= H // 8 and BS >= 2 and cap > 0 and smem <= 232448
        seen.add((pas, vl, tier))
        modes.add(mode)
    want = {(p, v, t) for p in ("fwd", "bwd") for v in ("0", "1") for t in ("smem", "l2")}
    assert seen == want, sorted(want - seen)
    assert modes == {"RNN_TANH", "RNN_RELU"}


def test_fused_paths_fall_back_to_the_module_forward():
    """forward_ln_sum of an Elman RNN is the unfused expression; the shell entry points refuse the mode"""
    torch.manual_seed(1)
    m = b200rnn.RNN(128, 128, nonlinearity="relu", batch_first=True).to(DEV)
    ln = torch.nn.LayerNorm(128).to(DEV)
    x = torch.randn(4, 9, 128, device=DEV)
    with torch.no_grad():
        got = m.forward_ln_sum(x, ln)
        want = m(ln(x))[0].sum(dim=1)
    assert torch.equal(got, want)
    from b200rnn.functional import rnn_forward_fused
    with pytest.raises(b200rnn.B200RNNError, match="mode"):
        rnn_forward_fused(x, m._flat_weights, m._config())


# ---- RNNCell ---------------------------------------------------------------------------------------------------------
BATCHES = (1, 7, 9, 130, 1024)
SHAPES = ((1, 1), (3, 5), (256, 256), (1024, 128), (40, 1000), (257, 129))


@pytest.mark.parametrize("nl", NONLIN)
@pytest.mark.parametrize("IH", SHAPES, ids=lambda s: f"I{s[0]}H{s[1]}")
@pytest.mark.parametrize("B", BATCHES)
def test_cell_forward_and_backward_against_float64(nl, IH, B):
    I, H = IH
    for bias, hx_given in ((True, True), (False, False), (True, False), (False, True)):
        torch.manual_seed(I + H)
        stock = torch.nn.RNNCell(I, H, bias=bias, nonlinearity=nl)
        mine = b200rnn.from_torch(stock).to(DEV)
        ref = stock.double()
        g = torch.Generator().manual_seed(1)
        x = torch.randn(B, I, generator=g)
        h = (torch.rand(B, H, generator=g) * 2 - 1) if hx_given else None
        w = torch.randn(B, H, generator=g, dtype=torch.float64)
        xm, xr = x.to(DEV).requires_grad_(True), x.double().requires_grad_(True)
        hm = h.to(DEV).requires_grad_(True) if hx_given else None
        hr = h.double().requires_grad_(True) if hx_given else None
        om, orf = mine(xm, hm), ref(xr, hr)
        if nl == "relu":  # a pre-activation within rounding of 0 may be on different sides of it in fp32 and float64:
            w = w * ((om > 0).cpu() == (orf > 0))  # such an output has no common derivative, and no weight here
        (om * w.to(DEV, torch.float32)).sum().backward()
        (orf * w).sum().backward()
        torch.cuda.synchronize()
        assert _out_err(nl, _np(om), _np(orf)) <= OUT_TOL
        assert _rel(_np(xm.grad), _np(xr.grad)) <= GRAD_RTOL
        if hx_given:
            assert _rel(_np(hm.grad), _np(hr.grad)) <= GRAD_RTOL
        for (n, pr), pm in zip(ref.named_parameters(), mine.parameters()):
            assert _rel(_np(pm.grad), _np(pr.grad)) <= GRAD_RTOL, n
        if B == 1:  # unbatched: the same step
            with torch.no_grad():
                o1 = mine(x[0].to(DEV), h[0].to(DEV) if hx_given else None)
            assert o1.shape == (H,) and torch.equal(o1, om[0].detach())


@pytest.mark.parametrize("nl", NONLIN)
def test_cell_tf32_mode_within_the_tf32_bound(nl):
    for I, H in ((256, 256), (257, 129), (40, 1000)):
        torch.manual_seed(H)
        stock = torch.nn.RNNCell(I, H, nonlinearity=nl)
        mine = b200rnn.from_torch(stock).to(DEV)
        g = torch.Generator().manual_seed(2)
        x, h = 2.0 * torch.randn(130, I, generator=g), torch.rand(130, H, generator=g) * 2 - 1
        with torch.no_grad(), _tf32(True):
            out = mine(x.to(DEV), h.to(DEV))
        w = [_np(p) for p in stock.parameters()]
        pre = _np(x) @ w[0].T + w[2] + w[3] + _np(h) @ w[1].T
        S = np.abs(_np(x)) @ np.abs(w[0]).T + np.abs(w[2]) + np.abs(w[3]) + np.abs(_np(h)) @ np.abs(w[1]).T
        want = np.tanh(pre) if nl == "tanh" else np.maximum(pre, 0.0)
        ratio = np.abs(_np(out) - want) / (KAPPA * U_TF32 * (S + 1.0))
        assert ratio.max() <= 1.0, ratio.max()
