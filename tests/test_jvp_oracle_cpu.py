"""CPU tests pinning the linearised steps of the oracle (oracle.rnn_numpy.gru_step_jvp / lstm_step_jvp / elman_step_jvp)
and their bound: each step equals float64 torch.func.jvp of the stock cell for every tangent group alone and all together,
an fp32 evaluation of the same step stays within KAPPA_T u S' in the saturated and large-input regimes, and, for the
Elman cell, one with TF32-rounded weights does not. For the GRU and LSTM the primal's share of S' (the saved gates' own
error bound times the tangent magnitudes it scales) dominates the bound - the fp32 evaluation sits ~1e-3 of it - and a
TF32-rounded operand stays inside it (measured 0.05 - 1.3 of it): the per-step test cannot tell TF32 from fp32 there, and
the free-running test of tests/test_gpu_jvp_numerics_f64.py, calibrated against stock fp32, is the one that does."""
import numpy as np
import pytest
import torch
from torch.func import functional_call, jvp

from oracle.rnn_numpy import elman_step_jvp, gru_step_jvp, lstm_step_jvp
from oracle.tf32 import round_tf32
from test_gpu_jvp_numerics_f64 import KAPPA_T

U32 = 2.0 ** -24
KINDS = ("gru", "lstm", "rnn_tanh", "rnn_relu")
# which tangents are non-zero: each group alone, then all of them
GROUPS = ("x", "h", "c", "weight_ih", "weight_hh", "bias", "all")
NAMES = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")


def _cell(kind, I, H, regime, seed=0):
    torch.manual_seed(seed)
    cell = {"gru": lambda: torch.nn.GRUCell(I, H), "lstm": lambda: torch.nn.LSTMCell(I, H),
            "rnn_tanh": lambda: torch.nn.RNNCell(I, H, nonlinearity="tanh"),
            "rnn_relu": lambda: torch.nn.RNNCell(I, H, nonlinearity="relu")}[kind]().double()
    g = torch.Generator().manual_seed(seed + 100)
    if regime == "saturated" and kind != "rnn_relu":
        with torch.no_grad():
            for n, p in cell.named_parameters():
                p.copy_(p * 4.0 if n.startswith("weight") else torch.rand(p.shape, generator=g, dtype=p.dtype) * 6 - 3)
    return cell


def _case(kind, group, regime, I=40, H=24, B=7, seed=0):
    """the cell, primal inputs and tangents (zero outside the group) in float64"""
    cell = _cell(kind, I, H, regime, seed)
    g = torch.Generator().manual_seed(seed + 1)
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    x = rnd(B, I) * {"default": 1.0, "saturated": 2.0, "large_input": 30.0}[regime]
    st = [torch.rand(B, H, generator=g, dtype=torch.float64) * 2 - 1] + ([rnd(B, H)] if kind == "lstm" else [])
    p = {n: t.detach() for n, t in cell.named_parameters()}
    on = lambda k: group in ("all", k)  # noqa: E731
    xd = rnd(B, I) if on("x") else torch.zeros(B, I, dtype=torch.float64)
    sd = [rnd(B, H) if on(k) else torch.zeros(B, H, dtype=torch.float64) for k in ("h", "c")[:len(st)]]
    pd = {n: rnd(*t.shape) if on(n) or (group == "bias" and n.startswith("bias")) else torch.zeros_like(t)
          for n, t in p.items()}
    return cell, p, x, st, pd, xd, sd


def _torch_jvp(kind, cell, p, x, st, pd, xd, sd):
    def f(p, x, *st):
        out = functional_call(cell, p, (x, tuple(st) if kind == "lstm" else st[0]))
        return out if kind == "lstm" else (out,)
    _, t = jvp(f, (p, x, *st), (pd, xd, *sd))
    return [v.numpy() for v in t]


def _oracle(kind, p, x, st, pd, xd, sd, dtype=np.float64):
    """the oracle's step; dtype float32 keeps the inputs exact and returns only the bound"""
    n = lambda t: t.numpy() if isinstance(t, torch.Tensor) else t  # noqa: E731
    w = [n(p[k]) for k in NAMES]
    wd = [n(pd[k]) for k in NAMES]
    if kind == "gru":
        return gru_step_jvp(n(x), n(st[0]), *w, n(xd), n(sd[0]), *wd)
    if kind == "lstm":
        return lstm_step_jvp(n(x), n(st[0]), n(st[1]), *w, n(xd), n(sd[0]), n(sd[1]), *wd)
    return elman_step_jvp(n(x), n(st[0]), *w, n(xd), n(sd[0]), *wd, nonlinearity=kind[4:])


@pytest.mark.parametrize("group", GROUPS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("regime", ["default", "saturated"])
def test_linearised_steps_equal_float64_torch_jvp_of_the_stock_cell(kind, group, regime):
    if group == "c" and kind != "lstm":
        pytest.skip("only the LSTM has a cell state")
    cell, p, x, st, pd, xd, sd = _case(kind, group, regime)
    want = _torch_jvp(kind, cell, p, x, st, pd, xd, sd)
    got = _oracle(kind, p, x, st, pd, xd, sd)
    outs = got[:2] if kind == "lstm" else got[:1]
    for a, b in zip(outs, want):
        assert np.abs(a - b).max() <= 1e-12 * max(1.0, np.abs(b).max()), (kind, group)
    assert any(np.abs(b).max() > 0 for b in want)


# ---- fp32 evaluation of the same step, to pin the bound ----------------------------------------------------------------

def _sig(v):
    return np.float32(1) / (np.float32(1) + np.exp(-v))


def _fp32_step(kind, p, x, st, pd, xd, sd, rnd=lambda a: a):
    """the linearised step in fp32 as the kernel orders it: primal gates, then the tangent pre-activations (x side, h
    side), the linearised cell at the fp32 gates. `rnd` rounds the weight operands (the TF32 mutant)"""
    f = lambda t: np.asarray(t, dtype=np.float32)  # noqa: E731
    w_ih, w_hh, b_ih, b_hh = (f(p[k]) for k in NAMES)
    wid, whd, bid, bhd = (f(pd[k]) for k in NAMES)
    x, xd = f(x), f(xd)
    h, hd = f(st[0]), f(sd[0])
    H = h.shape[1]
    ai = (f(xd) @ rnd(w_ih).T + x @ rnd(wid).T) + bid
    ah = (hd @ rnd(w_hh).T + h @ rnd(whd).T)
    if kind == "gru":
        gi, gh = x @ w_ih.T + b_ih, h @ w_hh.T + b_hh
        r, z = _sig(gi[:, :H] + gh[:, :H]), _sig(gi[:, H:2 * H] + gh[:, H:2 * H])
        hn = gh[:, 2 * H:]
        n = np.tanh(gi[:, 2 * H:] + r * hn)
        a = ai[:, :2 * H] + (ah[:, :2 * H] + bhd[:2 * H])
        ahn = ah[:, 2 * H:] + bhd[2 * H:]
        dr, dz = r * (1 - r) * a[:, :H], z * (1 - z) * a[:, H:]
        dn = (1 - n * n) * (ai[:, 2 * H:] + dr * hn + r * ahn)
        return [(1 - z) * dn + z * hd + dz * (h - n)]
    a = ai + (ah + bhd)
    pa = x @ w_ih.T + b_ih + h @ w_hh.T + b_hh
    if kind == "lstm":
        c, cd = f(st[1]), f(sd[1])
        i, fg, g, o = _sig(pa[:, :H]), _sig(pa[:, H:2 * H]), np.tanh(pa[:, 2 * H:3 * H]), _sig(pa[:, 3 * H:])
        c_new = fg * c + i * g
        di, df = i * (1 - i) * a[:, :H], fg * (1 - fg) * a[:, H:2 * H]
        dg, do = (1 - g * g) * a[:, 2 * H:3 * H], o * (1 - o) * a[:, 3 * H:]
        cdot = df * c + fg * cd + di * g + i * dg
        tc = np.tanh(c_new)
        return [do * tc + o * (1 - tc * tc) * cdot, cdot]
    if kind == "rnn_relu":
        return [np.where(pa > 0, a, np.float32(0))]
    hh = np.tanh(pa)
    return [(1 - hh * hh) * a]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("regime", ["saturated", "large_input"])
def test_fp32_step_within_the_bound_and_tf32_operands_beyond_it(kind, regime):
    """every element of an fp32 evaluation within KAPPA_T u S'; for the Elman cell, with the weights (and weight
    tangents) rounded to TF32, the worst element exceeds the bound at least 4 times over in the saturated regime (measured
    8 - 18 times; large_input: 1 - 12 times, not asserted)"""
    I, H, B = (1024 if regime == "large_input" else 256), 256, 16
    cell, p, x, st, pd, xd, sd = _case(kind, "all", regime, I=I, H=H, B=B)
    # the inputs the fp32 evaluation sees, exactly: the float64 reference starts from the same values
    q = lambda t: torch.from_numpy(np.asarray(t.numpy(), dtype=np.float32).astype(np.float64))  # noqa: E731
    p, pd = {k: q(v) for k, v in p.items()}, {k: q(v) for k, v in pd.items()}
    x, xd, st, sd = q(x), q(xd), [q(s) for s in st], [q(s) for s in sd]
    res = _oracle(kind, p, x, st, pd, xd, sd)
    want, bounds = (res[:2], res[2:]) if kind == "lstm" else (res[:1], res[1:])
    if kind == "rnn_relu":   # the precondition of the relu bound: no pre-activation within reach of its branch point
        pa = x.numpy() @ p["weight_ih"].numpy().T + st[0].numpy() @ p["weight_hh"].numpy().T
        keep = np.abs(pa + p["bias_ih"].numpy() + p["bias_hh"].numpy()) > 1e-3
    else:
        keep = True
    ratio = lambda got: max(float((np.abs(g - w) / (KAPPA_T * U32 * s))[keep].max())  # noqa: E731
                            for g, w, s in zip(got, want, bounds))
    ok = ratio(_fp32_step(kind, p, x, st, pd, xd, sd))
    bad = ratio(_fp32_step(kind, p, x, st, pd, xd, sd, rnd=lambda w: round_tf32(w).astype(np.float32)))
    assert ok <= 1.0, (kind, regime, ok)
    if kind.startswith("rnn") and regime == "saturated":
        assert bad > 4.0, (kind, regime, bad)
