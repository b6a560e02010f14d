"""GRU / LSTM at hidden sizes other than 128 / 256: the runtime-sized cluster kernels of csrc/rnn_anyh.cu.

Oracles: oracle/rnn_numpy.py in float64 and stock torch.nn.GRU / LSTM on CPU. Tolerances as DESIGN.md §2: outputs and
states 1e-5 absolute, gradients 1e-4 relative to the largest entry of each tensor. The per-step test holds each step of
the kernel's own trajectory to kappa * u * S (tests/test_gpu_numerics_f64.py) away from default init. Which config each
shape runs (cluster width C, batch rows BS, weight tier) is read from the B200RNN_DEBUG lines of a subprocess: every
instantiation (GRU / LSTM x fixed / ragged x shared-memory / L2 weights, forward and backward) is reached."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OUT_TOL = 1e-5
GRAD_RTOL = 1e-4
KAPPA = 24.0
U32 = 2.0 ** -24
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _abs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _np(t):
    return t.detach().cpu().double().numpy()


# kind, H, I, L, bidirectional, batch_first, B, T
CASES = [
    ("gru", 16, 7, 1, False, False, 3, 7),
    ("lstm", 16, 16, 2, True, True, 1, 1),
    ("gru", 48, 30, 2, True, True, 64, 7),
    ("lstm", 48, 33, 1, False, False, 3, 120),
    ("gru", 64, 40, 3, False, False, 128, 7),
    ("lstm", 64, 64, 2, True, False, 200, 7),
    ("gru", 96, 13, 1, True, True, 3, 120),
    ("lstm", 112, 50, 2, False, True, 64, 7),
    ("gru", 192, 64, 1, False, False, 200, 7),
    ("lstm", 192, 21, 1, True, True, 3, 1),
    ("gru", 320, 32, 2, False, False, 64, 7),
    ("lstm", 384, 64, 1, False, True, 128, 7),
    ("gru", 512, 64, 1, True, False, 64, 7),
    ("lstm", 512, 48, 1, False, False, 3, 120),
    ("gru", 768, 64, 1, False, True, 16, 7),
    ("lstm", 768, 32, 1, True, False, 3, 7),
    ("gru", 1024, 64, 1, False, False, 200, 7),
    ("lstm", 1024, 100, 2, False, True, 64, 1),
]


def _case_id(c):
    return f"{c[0]}{c[1]}_I{c[2]}_L{c[3]}_D{2 if c[4] else 1}_{'bf' if c[5] else 'tm'}_B{c[6]}_T{c[7]}"


@pytest.mark.parametrize("kind, H, I, L, bi, bf, B, T", CASES, ids=[_case_id(c) for c in CASES])
def test_matches_float64_and_torch(kind, H, I, L, bi, bf, B, T):
    """y, h_n, c_n, dx and every dW / db against float64 and against stock torch on CPU"""
    import b200rnn
    from oracle.rnn_numpy import NumpyRNN

    torch.manual_seed(H + L)
    ref = (torch.nn.GRU if kind == "gru" else torch.nn.LSTM)(I, H, num_layers=L, bidirectional=bi, batch_first=bf)
    mine = b200rnn.from_torch(ref).to(DEV).eval()
    g = torch.Generator().manual_seed(7)
    D = 2 if bi else 1
    shape = (B, T, I) if bf else (T, B, I)
    x = torch.randn(*shape, generator=g)
    yshape = (B, T, D * H) if bf else (T, B, D * H)
    wy = torch.randn(*yshape, generator=g)
    ws = [torch.randn(L * D, B, H, generator=g) for _ in range(1 if kind == "gru" else 2)]

    def run(model, dev):
        model.zero_grad(set_to_none=True)
        xx = x.clone().to(dev).requires_grad_(True)
        out = model(xx)
        states = out[1] if isinstance(out[1], tuple) else (out[1],)
        loss = (out[0] * wy.to(dev)).sum() + sum((s * w.to(dev)).sum() for s, w in zip(states, ws))
        loss.backward()
        return out[0], states, xx.grad, [p.grad for p in model.parameters()]

    y_m, s_m, dx_m, gp_m = run(mine, DEV)
    torch.cuda.synchronize()
    y_r, s_r, dx_r, gp_r = run(ref, "cpu")
    names = [n for n, _ in ref.named_parameters()]
    assert _abs(_np(y_m), _np(y_r)) <= OUT_TOL
    for a, b in zip(s_m, s_r):
        assert _abs(_np(a), _np(b)) <= OUT_TOL
    assert _rel(_np(dx_m), _np(dx_r)) <= GRAD_RTOL
    for n, a, b in zip(names, gp_m, gp_r):
        assert _rel(_np(a), _np(b)) <= GRAD_RTOL, n

    # float64, time-major
    orc = NumpyRNN(kind, [p.detach().double().numpy() for p in ref.parameters()], L, bi)
    xt = x.double().numpy() if not bf else x.double().numpy().transpose(1, 0, 2)
    res = orc.forward(xt)
    y64 = res[0] if not bf else res[0].transpose(1, 0, 2)
    assert _abs(_np(y_m), y64) <= OUT_TOL
    for a, b in zip(s_m, res[1:]):
        assert _abs(_np(a), b) <= OUT_TOL
    wyt = wy.double().numpy() if not bf else wy.double().numpy().transpose(1, 0, 2)
    dx64, dps = orc.backward(wyt, *[w.double().numpy() for w in ws])
    dx64 = dx64 if not bf else dx64.transpose(1, 0, 2)
    assert _rel(_np(dx_m), dx64) <= GRAD_RTOL
    for n, a, b in zip(names, gp_m, dps):
        assert _rel(_np(a), b) <= GRAD_RTOL, n


@pytest.mark.parametrize("kind, H, B", [("gru", 64, 16), ("gru", 384, 5), ("gru", 1024, 3)])
def test_gru_per_step_bound_at_t120_non_default_init(kind, H, B):
    """Each step of a T = 120 launch, recomputed in float64 from the kernel's own h_{t-1} (its previous output), within
    KAPPA * u * S; weights at 3x the default init range and inputs x4, so that the gates saturate"""
    import b200rnn
    from oracle.rnn_numpy import gru_step

    T, I = 120, 40
    torch.manual_seed(H)
    m = b200rnn.GRU(I, H).to(DEV).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(3.0)
    x = 4.0 * torch.randn(T, B, I, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        y = _np(m(x.to(DEV))[0])
    w = [p.detach().double().cpu().numpy() for p in m.parameters()]
    worst, h = 0.0, np.zeros((B, H))
    for t in range(T):
        want, S = gru_step(x[t].double().numpy(), h, *w)
        worst = max(worst, float((np.abs(y[t] - want) / (KAPPA * U32 * S)).max()))
        h = y[t]
    print(f"GRU-{H} B{B}: worst per-step err / bound = {worst:.3f}")
    assert worst <= 1.0


@pytest.mark.parametrize("H", [48, 384, 768])
def test_lstm_per_step_bound_non_default_init(H):
    """LSTM: 120 one-step launches chained through hx, each recomputed in float64 from the kernel's (h, c) before it;
    h and c within KAPPA * u * S. Weights 3x the default range, inputs x4."""
    import b200rnn
    from oracle.rnn_numpy import lstm_step

    T, B, I = 120, 6, 24
    torch.manual_seed(H)
    m = b200rnn.LSTM(I, H).to(DEV).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(3.0)
    x = 4.0 * torch.randn(T, B, I, generator=torch.Generator().manual_seed(2))
    w = [p.detach().double().cpu().numpy() for p in m.parameters()]
    h = torch.zeros(1, B, H, device=DEV)
    c = torch.zeros(1, B, H, device=DEV)
    worst = 0.0
    with torch.no_grad():
        for t in range(T):
            _, (h1, c1) = m(x[t:t + 1].to(DEV), (h, c))
            want_h, want_c, S_h, S_c = lstm_step(x[t].double().numpy(), _np(h[0]), _np(c[0]), *w)
            worst = max(worst, float((np.abs(_np(h1[0]) - want_h) / (KAPPA * U32 * S_h)).max()),
                        float((np.abs(_np(c1[0]) - want_c) / (KAPPA * U32 * S_c)).max()))
            h, c = h1, c1
    print(f"LSTM-{H}: worst per-step err / bound = {worst:.3f}")
    assert worst <= 1.0


def _lengths(B, T, seed=5):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, T + 1, (B,), generator=g)
    lens[: B // 4] = torch.randint(1, 4, (B // 4,), generator=g)  # skewed: a quarter of very short rows
    lens[B // 2] = T
    return lens


@pytest.mark.parametrize("kind, H, B, T, bi, hx, hx_grad", [
    ("gru", 96, 64, 40, False, False, False),
    ("lstm", 48, 37, 30, True, True, True),
    ("gru", 512, 20, 25, True, True, False),     # shared-memory tier, ragged, reverse direction
    ("lstm", 768, 19, 20, False, True, True),    # L2 tier, ragged
    ("gru", 1024, 9, 12, True, False, False),
    ("lstm", 464, 13, 9, True, True, True),      # uneven slices: CTAs of 24 and 32 units
    ("gru", 1008, 6, 8, False, True, False),
])
def test_packed_sequence_and_hx(kind, H, B, T, bi, hx, hx_grad):
    """PackedSequence with skewed lengths, with and without an initial state, with and without dh_0 / dc_0"""
    import b200rnn

    I, L = 24, 2
    torch.manual_seed(3)
    ref = (torch.nn.GRU if kind == "gru" else torch.nn.LSTM)(I, H, num_layers=L, bidirectional=bi, batch_first=True)
    mine = b200rnn.from_torch(ref).to(DEV)
    D = 2 if bi else 1
    g = torch.Generator().manual_seed(4)
    x = torch.randn(B, T, I, generator=g)
    lens = _lengths(B, T)
    h0 = [0.5 * torch.randn(L * D, B, H, generator=g) for _ in range(1 if kind == "gru" else 2)]
    wy = torch.randn(B, T, D * H, generator=g)
    ws = [torch.randn(L * D, B, H, generator=g) for _ in h0]

    def run(model, dev):
        model.zero_grad(set_to_none=True)
        xx = x.clone().to(dev).requires_grad_(True)
        hh = [s.clone().to(dev).requires_grad_(hx_grad) for s in h0]
        packed = pack_padded_sequence(xx, lens, batch_first=True, enforce_sorted=False)
        state = None if not hx else (hh[0] if kind == "gru" else tuple(hh))
        out = model(packed, state)
        y = pad_packed_sequence(out[0], batch_first=True, total_length=T)[0]
        states = out[1] if isinstance(out[1], tuple) else (out[1],)
        loss = (y * wy.to(dev)).sum() + sum((s * w.to(dev)).sum() for s, w in zip(states, ws))
        loss.backward()
        return y, states, xx.grad, [p.grad for p in model.parameters()], [s.grad for s in hh]

    m, r = run(mine, DEV), run(ref, "cpu")
    assert _abs(_np(m[0]), _np(r[0])) <= OUT_TOL
    for a, b in zip(m[1], r[1]):
        assert _abs(_np(a), _np(b)) <= OUT_TOL
    assert _rel(_np(m[2]), _np(r[2])) <= GRAD_RTOL
    for a, b in zip(m[3], r[3]):
        assert _rel(_np(a), _np(b)) <= GRAD_RTOL
    for a, b in zip(m[4], r[4]):
        assert (a is None) == (b is None)
        if a is not None:
            assert _rel(_np(a), _np(b)) <= GRAD_RTOL


@pytest.mark.parametrize("kind, H", [("gru", 64), ("lstm", 320)])
def test_unbatched_input(kind, H):
    import b200rnn

    torch.manual_seed(8)
    ref = (torch.nn.GRU if kind == "gru" else torch.nn.LSTM)(20, H, num_layers=2, bidirectional=True)
    mine = b200rnn.from_torch(ref).to(DEV)
    x = torch.randn(9, 20)
    xm, xr = x.to(DEV).requires_grad_(True), x.clone().requires_grad_(True)
    ym, yr = mine(xm), ref(xr)
    assert ym[0].shape == yr[0].shape
    assert _abs(_np(ym[0]), _np(yr[0])) <= OUT_TOL
    ym[0].sum().backward()
    yr[0].sum().backward()
    assert _rel(_np(xm.grad), _np(xr.grad)) <= GRAD_RTOL


@pytest.mark.parametrize("kind, H", [("gru", 64), ("lstm", 96)])
def test_dropout_masks_of_forward_and_backward_agree(kind, H):
    """Train mode, p = 0.5, one step of one sequence: the units whose dW_ih_l1 column is zero are the ones the dropout
    zeroed; stock layer 1 on h0 * mask / (1 - p) reproduces the output (forward mask) and dx (backward mask)"""
    import b200rnn

    p = 0.5
    torch.manual_seed(6)
    cls = b200rnn.GRU if kind == "gru" else b200rnn.LSTM
    m = cls(32, H, num_layers=2, dropout=p, bidirectional=True).to(DEV).train()
    stock = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    layers = [stock(32 if i == 0 else 2 * H, H, bidirectional=True) for i in range(2)]
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
    frac = 1.0 - kept.float().mean().item()
    assert 0.2 < frac < 0.8, frac
    xr = x.clone().requires_grad_(True)
    h0 = layers[0](xr)[0]
    y_check = layers[1](h0 * kept / (1 - p))[0]
    (y_check * dy).sum().backward()
    assert _abs(_np(y), _np(y_check)) <= OUT_TOL
    assert _rel(_np(xm.grad), _np(xr.grad)) <= GRAD_RTOL


@pytest.mark.parametrize("kind, H, B", [("gru", 384, 24), ("lstm", 1024, 8)])
def test_tf32_mode_meets_the_emulation_bounds(kind, H, B):
    """torch's "tf32" matmul precision: the input projection and the gradient GEMMs go single-pass TF32 (I = 256 and
    G*H, H multiples of 128 put every GEMM on the tensor cores); the runtime-sized recurrence stays fp32.
    oracle/tf32.py rounds exactly those operands."""
    import b200rnn
    from b200rnn.functional import rnn_forward
    from oracle.tf32 import Tf32RNN

    T, I, L = 30, 256, 1
    torch.manual_seed(0)
    ref = (torch.nn.GRU if kind == "gru" else torch.nn.LSTM)(I, H, num_layers=L)
    mine = b200rnn.from_torch(ref).to(DEV).eval()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(T, B, I, generator=g)
    xm = x.to(DEV).requires_grad_(True)
    saved = (torch.backends.fp32_precision, torch.backends.cuda.matmul.fp32_precision)
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        cfg = mine._config()
        assert cfg.tf32
        out = rnn_forward(xm, mine._flat_weights, cfg)
    finally:
        torch.backends.fp32_precision, torch.backends.cuda.matmul.fp32_precision = saved
    states = out[1:]
    dy = torch.randn(out[0].shape, generator=g)
    dstates = [torch.randn(s.shape, generator=g) for s in states]
    loss = (out[0] * dy.to(DEV)).sum() + sum((s * d.to(DEV)).sum() for s, d in zip(states, dstates))
    loss.backward()
    torch.cuda.synchronize()
    orc = Tf32RNN(kind, [p.detach().double().numpy() for p in ref.parameters()], L, False, rec_round=False)
    res = orc.forward(x.double().numpy(), None, [_np(out[0])])
    assert _abs(_np(out[0]), res[0]) <= OUT_TOL
    for s, r in zip(states, res[1:]):
        assert _abs(_np(s), r) <= OUT_TOL
    dx, dps = orc.backward(dy.double().numpy(), *[d.double().numpy() for d in dstates])
    assert _rel(_np(xm.grad), dx) <= GRAD_RTOL
    for (n, _), p, d in zip(ref.named_parameters(), mine._flat_weights, dps):
        assert _rel(_np(p.grad), d) <= GRAD_RTOL, n


@pytest.mark.parametrize("kind, H, B, bi", [("gru", 96, 40, True), ("lstm", 768, 12, False)])
def test_cuda_graph_replay_is_bitwise_eager_and_runs_repeat(kind, H, B, bi):
    import b200rnn

    T, I = 20, 48
    torch.manual_seed(9)
    mine = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(I, H, num_layers=2, bidirectional=bi).to(DEV)
    D = 2 if bi else 1
    g = torch.Generator().manual_seed(3)
    x = torch.randn(T, B, I, generator=g).to(DEV)
    h0 = (0.5 * torch.randn(2 * D, B, H, generator=g)).to(DEV).requires_grad_(True)
    c0 = (0.5 * torch.randn(2 * D, B, H, generator=g)).to(DEV)
    wy = torch.randn(T, B, D * H, generator=g).to(DEV)

    def step():
        y, s = mine(x, h0 if kind == "gru" else (h0, c0))
        hn = s if kind == "gru" else s[0]
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
shapes = [("gru", 512, 64), ("lstm", 384, 64), ("gru", 1024, 8), ("lstm", 1024, 8), ("gru", 64, 200),
          ("gru", 256, 16), ("lstm", 128, 24)]
for kind, H, B in shapes:
    for ragged in (False, True):
        torch.manual_seed(0)
        m = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(16, H).cuda()
        x = torch.randn(5, B, 16, device="cuda", requires_grad=True)
        print("SHAPE", kind, H, B, int(ragged), file=sys.stderr, flush=True)
        if ragged:
            lens = torch.arange(B) % 5 + 1
            y = m(pack_padded_sequence(x, lens, enforce_sorted=False))[0].data
        else:
            y = m(x)[0]
        y.sum().backward()
        torch.cuda.synchronize()
"""


def _dispatch_lines():
    env = dict(os.environ, B200RNN_DEBUG="1")
    r = subprocess.run([sys.executable, "-c", _DISPATCH], capture_output=True, text=True, env=env,
                       cwd=os.path.join(ROOT, "icassp2022-depression_b200"), timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr.splitlines()


def test_dispatch_reaches_every_instantiation_and_both_tiers():
    lines = _dispatch_lines()
    pat = re.compile(r"\[b200rnn\] (fwd|bwd) anyh cfg (GRU|LSTM) VL=(\d) H=(\d+) C=(\d+) BS=(\d+) tier=(smem|l2): "
                     r"need (\d+) clusters, capacity (\d+), smem (\d+)")
    seen = set()
    for ln in lines:
        mt = pat.search(ln)
        if not mt:
            continue
        pas, kind, vl, H, C, BS, tier, need, cap, smem = mt.groups()
        H, C, BS, need, cap, smem = map(int, (H, C, BS, need, cap, smem))
        assert H not in (128, 256)
        assert C in (2, 4, 8, 16) and (H // C) % 8 == 0 and BS >= 2 and cap > 0 and smem <= 232448
        seen.add((pas, kind, vl, tier))
    want = {(p, k, v, t) for p in ("fwd", "bwd") for k in ("GRU", "LSTM") for v in ("0", "1") for t in ("smem", "l2")}
    assert seen == want, sorted(want - seen)
    # 128 / 256 keep their fixed configs and print the lines they printed before (the capacity is the device's)
    fixed = {
        "gru 256 16": ["fwd cfg C=4 BS=2 KL=16 UPL=8 RG=0 PB=0: need 8 clusters, capacity CAP, smem 200960",
                       "bwd cfg C=4 BS=2 KL=16 UPL=8 RG=0: need 8 clusters, capacity CAP, smem 209152"],
        "lstm 128 24": ["fwd cfg C=2 BS=4 KL=16 UPL=4 RG=1 PB=0: need 6 clusters, capacity CAP, smem 102656",
                        "bwd cfg C=2 BS=4 KL=32 UPL=8 RG=1: need 6 clusters, capacity CAP, smem 114944"],
    }
    text = "\n".join(lines)
    checked = 0
    for blk in text.split("SHAPE ")[1:]:
        key = " ".join(blk.split()[:3])
        if key in fixed:
            got = [re.sub(r"capacity \d+", "capacity CAP", ln.split("[b200rnn] ", 1)[1])
                   for ln in blk.splitlines() if re.search(r"\[b200rnn\] (fwd|bwd) .*cfg", ln)]
            assert got == fixed[key], (key, got)
            checked += 1
    assert checked == 4


def test_fused_entry_points_reject_other_hidden_sizes():
    import b200rnn
    from b200rnn import _lib
    from b200rnn.functional import rnn_forward_fused

    m = b200rnn.GRU(128, 64, batch_first=True).to(DEV)
    x = torch.randn(2, 3, 128, device=DEV)
    with torch.no_grad(), pytest.raises(_lib.B200RNNError, match="hidden_size"):
        rnn_forward_fused(x, m._flat_weights, m._config(), m._rng_state, None, None, 1e-5, pool_sum=True)
    # forward_ln_sum takes the unfused expression at H = 64 and matches it
    ln = torch.nn.LayerNorm(128).to(DEV)
    with torch.no_grad():
        got = m.forward_ln_sum(x, ln)
        want = m(ln(x))[0].sum(dim=1)
    assert torch.equal(got, want)


@pytest.mark.parametrize("H", [64, 512])
def test_model_classes_after_install_match_reference_shells(H):
    """AudioBiLSTM / TextBiLSTM built with hidden_dims 64 and 512 after install(): forward + backward against the
    oracle/ref_models.py shells on stock torch (T kept small: attention_pool_bwd holds T*H in one CTA)"""
    import b200rnn
    from oracle import ref_models

    cfg = dict(embedding_size=40, hidden_dims=H, dropout=0.0, rnn_layers=2, num_classes=2, bidirectional=True)
    for name, ref_cls, T in (("AudioBiLSTM", ref_models.RefAudio, 12), ("TextBiLSTM", ref_models.RefText, 10)):
        torch.manual_seed(H)
        ref = ref_cls(cfg).eval()
        b200rnn.install()
        try:
            mine = getattr(b200rnn, name)(cfg)
        finally:
            b200rnn.uninstall()
        mine.load_state_dict(ref.state_dict())
        mine = mine.to(DEV).eval()
        x = torch.randn(3, T, 40, generator=torch.Generator().manual_seed(2))
        xr, xm = x.clone().requires_grad_(True), x.to(DEV).requires_grad_(True)
        out_r, out_m = ref(xr), mine(xm)
        w = torch.randn(out_r.shape, generator=torch.Generator().manual_seed(3))
        (out_r * w).sum().backward()
        (out_m * w.to(DEV)).sum().backward()
        assert _abs(_np(out_m), _np(out_r)) <= 1e-4, name
        assert _rel(_np(xm.grad), _np(xr.grad)) <= GRAD_RTOL, name
        pm = dict(mine.named_parameters())
        for n, p in ref.named_parameters():
            if p.grad is not None:
                assert _rel(_np(pm[n].grad), _np(p.grad)) <= GRAD_RTOL, (name, n)


@pytest.mark.parametrize("H", list(range(16, 1025, 16)))
def test_every_multiple_of_16_runs_forward_and_backward(H):
    """Every accepted hidden size runs, GRU and LSTM, bidirectional, forward and backward, against float64. Sizes whose
    H / 8 groups do not split evenly over the cluster (272, 464, 544, 1008, ...) give the CTAs unequal slices."""
    import b200rnn
    from oracle.rnn_numpy import NumpyRNN

    T, B, I = 5, 3, 24
    for kind in ("gru", "lstm"):
        torch.manual_seed(H)
        ref = (torch.nn.GRU if kind == "gru" else torch.nn.LSTM)(I, H, bidirectional=True)
        mine = b200rnn.from_torch(ref).to(DEV)
        g = torch.Generator().manual_seed(H + 1)
        x = torch.randn(T, B, I, generator=g)
        wy = torch.randn(T, B, 2 * H, generator=g)
        xm = x.to(DEV).requires_grad_(True)
        out = mine(xm)
        (out[0] * wy.to(DEV)).sum().backward()
        orc = NumpyRNN(kind, [p.detach().double().numpy() for p in ref.parameters()], 1, True)
        res = orc.forward(x.double().numpy())
        assert _abs(_np(out[0]), res[0]) <= OUT_TOL, kind
        dx64, dps = orc.backward(wy.double().numpy())
        assert _rel(_np(xm.grad), dx64) <= GRAD_RTOL, kind
        for (n, _), p, d in zip(ref.named_parameters(), mine.parameters(), dps):
            assert _rel(_np(p.grad), d) <= GRAD_RTOL, (kind, n)
