"""Every recurrence config against float64, away from default init.

The other GPU tests compare with stock torch in fp32 at default init, where no gate saturates and a fixed 1e-5 fits a
TF32-accurate contraction as well as an fp32-accurate one. Here every entry of both plan tables (csrc/rnn_rec.cu
plan_rec_fwd / plan_rec_bwd), fixed-length and ragged, runs in four weight / input regimes:

  default       torch's init, x ~ N(0, 1)
  saturated     weights x4, biases U(-3, 3), LSTM forget bias +3, x ~ N(0, 2^2)
  large_input   I = 1024, x x30 (the text encoder's input-projection magnitude)
  small_signal  x and biases x1e-3, so |h| ~ 1e-4

Per-step test (teacher forced). Each step of the kernel's own trajectory is recomputed in float64 from the kernel's own
previous state (oracle.rnn_numpy.gru_step / lstm_step), and every element must satisfy

    |h_kernel - step64(h_prev_kernel)| <= KAPPA * u * S

S = 1 + the sum of the absolute values of the terms the element is computed from (rnn_numpy.py). u = 2^-24 for the fp32
FFMA, 3xTF32 and fp16-pair contractions, 2^-11 in TF32 mode. KAPPA counts rounding stages, not measurements:
  - each pre-activation is one sum of I + H + 2 terms, reached by at most 4 roundings at the sum's own magnitude
    (the input-projection accumulator, its bias, the recurrent accumulator, the combine) plus the error of the
    accumulation itself. An accumulation chain of depth d errs by sqrt(d) u |terms| with high probability when the
    roundings are independent (Higham & Mary, SIAM J. Sci. Comput. 41(5), 2019); the longest chain in the library is
    the input-projection GEMM at I = 1024 with k-blocks of 8 (d = 128), sqrt(128) < 12, so 16 stages in all;
  - each activation adds its absolute error (common.cuh: ~1e-7 < 2u) and the cell update four more roundings
    (GRU: r * hn, (1 - z) n, z h, the add; LSTM: f c, i g, the add, o tanh(c)): 8 stages in all;
  - the gate derivatives are at most 1, so nothing is amplified within a step.
KAPPA = 16 + 8 = 24. A contraction that loses its hi/lo correction term errs by 2^-12 relative per product, ~2^12 / sqrt(K)
times u S over K terms: 2^8 u S at K = 256, ten times the bound.

Free-running test. Whole sequences and every gradient against float64 autograd (stock nn.GRU / nn.LSTM, .double(), CPU),
normwise per tensor, bounded by what stock torch in fp32 on CPU gets on the same inputs:

    err_kernel <= 4 * err_torch32 + 1e-6        (TF32 mode: err_torch32 scaled by 2^13 = u_tf32 / u_fp32)

Also: non-finite padding (NaN, +Inf, -Inf past each length) changes no output, state or gradient and reaches no padded
row, through the module path and through the C ABI with the LayerNorm prologue; and a NaN in one valid (t, b) reaches
exactly that row from that step on (forward in time, backward in time in the reverse half of a bidirectional layer).

B200RNN_NUMERICS_RECORD=<path> writes the per-config ratios (max err / bound, err_kernel / err_torch32) as JSON."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
KAPPA = 24.0
U32, U_TF32 = 2.0 ** -24, 2.0 ** -11
RECORDS = {}

# name -> kind, I, H, B, bidirectional, proj_size, contraction ("fp32", "tf32" or "f16" = the no-grad fused forward);
# the batch sizes pick the config on an H100 (66 two-CTA, 30 four-CTA, 15 eight-CTA co-resident clusters, DESIGN.md)
CONFIGS = {
    "gru256_bs2": ("gru", 256, 256, 16, False, 0, "fp32"),
    "gru256_bs4": ("gru", 256, 256, 64, False, 0, "fp32"),
    "gru256_tc8_3xtf32": ("gru", 256, 256, 128, False, 0, "fp32"),
    "gru256_tc8_tf32": ("gru", 256, 256, 128, False, 0, "tf32"),
    "gru256_tc8_f16pair": ("gru", 256, 256, 128, False, 0, "f16"),
    "gru128": ("gru", 40, 128, 64, False, 0, "fp32"),
    "gru128_wide": ("gru", 40, 128, 272, False, 0, "fp32"),
    "bilstm256": ("lstm", 256, 256, 32, True, 0, "fp32"),
    "bilstm256_wide": ("lstm", 256, 256, 64, True, 0, "fp32"),
    "bilstm128": ("lstm", 256, 128, 16, True, 0, "fp32"),
    "bilstm128_wide": ("lstm", 256, 128, 136, True, 0, "fp32"),
    "bilstmp_h128_p32": ("lstm", 256, 128, 16, True, 32, "fp32"),
    "bilstmp_h128_p64": ("lstm", 256, 128, 16, True, 64, "fp32"),
    "bilstmp_h256_p64": ("lstm", 256, 256, 16, True, 64, "fp32"),
    "bilstmp_h256_p128": ("lstm", 256, 256, 16, True, 128, "fp32"),
    "bilstm128_tcl8_f16pair": ("lstm", 256, 128, 128, True, 0, "f16"),
}
# the config line each entry must run (B200RNN_DEBUG), forward and backward
FWD_LINE = {
    "gru256_bs2": "fwd cfg C=4 BS=2 KL=16 UPL=8 RG=0 PB=0",
    "gru256_bs4": "fwd cfg C=4 BS=4 KL=16 UPL=4 RG=1 PB=1",
    "gru256_tc8_3xtf32": "fwd cfg tc8 C=4 BS=8 mma.sync 3xTF32",
    "gru256_tc8_tf32": "fwd cfg tc8 C=4 BS=8 mma.sync TF32",
    "gru256_tc8_f16pair": "fwd cfg tc8 C=4 BS=8 mma.sync f16x3",
    "gru128": "fwd cfg C=2 BS=4 KL=16 UPL=4 RG=1 PB=0",
    "gru128_wide": "fwd cfg C=4 BS=8 KL=32 UPL=4 RG=1 PB=0",
    "bilstm256": "fwd cfg C=4 BS=4 KL=16 UPL=4 RG=1 PB=0",
    "bilstm256_wide": "fwd cfg C=8 BS=8 KL=16 UPL=2 RG=1 PB=0",
    "bilstm128": "fwd cfg C=2 BS=4 KL=16 UPL=4 RG=1 PB=0",
    "bilstm128_wide": "fwd cfg C=4 BS=8 KL=16 UPL=2 RG=1 PB=0",
    "bilstmp_h128_p32": "fwd proj cfg C=2 BS=4 P=32",
    "bilstmp_h128_p64": "fwd proj cfg C=2 BS=4 P=64",
    "bilstmp_h256_p64": "fwd proj cfg C=4 BS=8 P=64",
    "bilstmp_h256_p128": "fwd proj cfg C=4 BS=8 P=128",
    "bilstm128_tcl8_f16pair": "fwd cfg tcl8 C=2 BS=8 mma.sync f16x3",
}
BWD_LINE = {
    "gru256_bs2": "bwd cfg C=4 BS=2 KL=16 UPL=8 RG=0",
    "gru256_bs4": "bwd cfg C=4 BS=4 KL=32 UPL=8 RG=1",
    "gru256_tc8_3xtf32": "bwd cfg C=8 BS=8 KL=32 UPL=4 RG=1",
    "gru256_tc8_tf32": "bwd cfg C=8 BS=8 KL=32 UPL=4 RG=1",
    "gru128": "bwd cfg C=2 BS=4 KL=32 UPL=8 RG=1",
    "gru128_wide": "bwd cfg C=4 BS=8 KL=32 UPL=4 RG=1",
    "bilstm256": "bwd cfg C=4 BS=4 KL=32 UPL=8 RG=1",
    "bilstm256_wide": "bwd cfg C=8 BS=8 KL=32 UPL=4 RG=1",
    "bilstm128": "bwd cfg C=2 BS=4 KL=32 UPL=8 RG=1",
    "bilstm128_wide": "bwd cfg C=4 BS=8 KL=32 UPL=4 RG=1",
    "bilstmp_h128_p32": "bwd proj cfg C=2 BS=4 P=32",
    "bilstmp_h128_p64": "bwd proj cfg C=2 BS=4 P=64",
    "bilstmp_h256_p64": "bwd proj cfg C=4 BS=8 P=64",
    "bilstmp_h256_p128": "bwd proj cfg C=4 BS=8 P=128",
}
# plan_rec_fwd: 5 GRU-256 contractions, 2 GRU-128, 2 LSTM-256, 3 LSTM-128 (FFMA narrow and wide, fp16-pair tcl8),
# 4 projected; plan_rec_bwd: 3 + 2 + 2 + 2 + 4
N_FWD_ENTRIES, N_BWD_ENTRIES = 16, 13
REGIMES = ("default", "saturated", "large_input", "small_signal")


@pytest.fixture(scope="module", autouse=True)
def _record():
    yield
    path = os.environ.get("B200RNN_NUMERICS_RECORD")
    if path and RECORDS:
        with open(path, "w") as f:
            json.dump(RECORDS, f, indent=1, sort_keys=True)
            f.write("\n")


def _record_ratio(kind, name, regime, key, value):
    RECORDS.setdefault(kind, {}).setdefault(name, {}).setdefault(regime, {})[key] = float(value)


# ---- models and inputs ------------------------------------------------------------------------------------------------

def _torch_model(kind, I, H, bi, P, regime, seed=0):
    """stock torch module (fp32, CPU) with the regime's weights"""
    torch.manual_seed(seed)
    cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    ref = cls(I, H, num_layers=1, bidirectional=bi, **({"proj_size": P} if P else {}))
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for n, p in ref.named_parameters():
            if regime == "saturated":
                if n.startswith("bias"):
                    p.copy_(torch.rand(p.shape, generator=g) * 6 - 3)
                    if kind == "lstm" and n.startswith("bias_ih"):
                        p[H:2 * H] += 3.0   # forget gate
                else:
                    p.mul_(4.0)
            elif regime == "small_signal" and n.startswith("bias"):
                p.mul_(1e-3)
    return ref


def _input(regime, T, B, I, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, B, I, generator=g)
    return x * {"default": 1.0, "saturated": 2.0, "large_input": 30.0, "small_signal": 1e-3}[regime]


def _shape(name, regime):
    kind, I, H, B, bi, P, mode = CONFIGS[name]
    if regime == "large_input":
        I = 1024
    return kind, I, H, B, bi, P, mode


def _ragged_lengths(B, T, seed=3):
    lens = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(seed))
    lens[0], lens[1 % B], lens[2 % B] = T, 0, 1
    return lens


def _cfg(mine, mode):
    cfg = mine._config()
    cfg.tf32 = mode == "tf32"
    return cfg


def _forward(mine, mode, x_tm, lengths=None, hx=None):
    """y [T,B,D*HO], h_n [, c_n] of the library on x_tm (time-major, on the device)"""
    from b200rnn.functional import rnn_forward, rnn_forward_fused

    with torch.no_grad():
        if mode == "f16":   # no initial state, fixed length
            return rnn_forward_fused(x_tm, mine._flat_weights, _cfg(mine, mode))
        return rnn_forward(x_tm, mine._flat_weights, _cfg(mine, mode), lengths=lengths, hx=hx)


def _f64_weights(ref, d):
    sfx = "_l0" + ("_reverse" if d else "")
    w = [getattr(ref, n + sfx).detach().double().numpy() for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    return w + ([getattr(ref, "weight_hr" + sfx).detach().double().numpy()] if ref.proj_size else [])


# ---- per-step, teacher forced -----------------------------------------------------------------------------------------

def _per_step(name, regime, ragged, T):
    from b200rnn import from_torch
    from oracle.rnn_numpy import gru_step, lstm_step

    kind, I, H, B, bi, P, mode = _shape(name, regime)
    if mode == "f16" and ragged:
        pytest.skip("the fp16-pair forward is the no-grad fused entry; its ragged form runs in test_gpu_h16_fwd.py and "
                    "test_gpu_lstm_h16_fwd.py")
    ref = _torch_model(kind, I, H, bi, P, regime)
    mine = from_torch(ref).to(DEV)
    x = _input(regime, T, B, I)
    lens = _ragged_lengths(B, T) if ragged else None
    u = U_TF32 if mode == "tf32" else U32
    D, HO = (2 if bi else 1), (P or H)
    worst = 0.0
    x64 = x.double().numpy()
    if kind == "gru":   # one call: the trajectory is y itself
        y = _forward(mine, mode, x.to(DEV), lens)[0].cpu().double().numpy()
        w = _f64_weights(ref, 0)
        h_prev = np.zeros((B, H))
        for t in range(T):
            live = np.ones(B, bool) if lens is None else (t < lens.numpy())
            h64, S = gru_step(x64[t], h_prev, *w)
            err = np.abs(y[t] - h64)[live]
            worst = max(worst, (err / (KAPPA * u * S[live])).max(initial=0.0))
            assert (y[t][~live] == 0).all(), (name, t)
            h_prev = np.where(live[:, None], y[t], h_prev)
    elif mode == "f16":   # the no-grad fused entry takes no initial state: each step's state from a prefix run
        # (forward direction: x[:t]) and a suffix run (reverse direction: x[T-t:]), whose outputs must be bitwise the
        # full run's
        y_full = _forward(mine, mode, x.to(DEV))[0].cpu()
        ws = [_f64_weights(ref, d) for d in range(D)]
        prev = [(np.zeros((B, H)), np.zeros((B, H))) for _ in range(D)]
        for t in range(1, T + 1):
            runs = [_forward(mine, mode, x[:t].to(DEV))] + ([_forward(mine, mode, x[T - t:].to(DEV))] if bi else [])
            assert torch.equal(runs[0][0].cpu()[:, :, :H], y_full[:t, :, :H]), (name, t)
            if bi:
                assert torch.equal(runs[1][0].cpu()[:, :, H:], y_full[T - t:, :, H:]), (name, t)
            for d in range(D):
                hn, cn = (a[d].cpu().double().numpy() for a in runs[d][1:3])
                hp, cp = prev[d]
                h64, c64, S_h, S_c = lstm_step(x64[t - 1] if d == 0 else x64[T - t], hp, cp, *ws[d][:4])
                for got, want, S in ((hn, h64, S_h), (cn, c64, S_c)):
                    worst = max(worst, (np.abs(got - want) / (KAPPA * u * S)).max())
                prev[d] = (hn, cn)
    else:   # LSTM / LSTMP: chained one-step calls through hx, which return the cell state as well
        h = torch.zeros(D, B, HO, device=DEV)
        c = torch.zeros(D, B, H, device=DEV)
        ws = [_f64_weights(ref, d) for d in range(D)]
        for t in range(T):
            live = np.ones(B, bool) if lens is None else (t < lens.numpy())
            step_len = None if lens is None else torch.from_numpy(live.astype(np.int32))
            _, h1, c1 = _forward(mine, mode, x[t:t + 1].to(DEV), step_len, (h, c))
            hp, cp, hn, cn = (a.cpu().double().numpy() for a in (h, c, h1, c1))
            for d in range(D):
                w_ih, w_hh, b_ih, b_hh, *w_hr = ws[d]
                h64, c64, S_h, S_c = lstm_step(x64[t], hp[d], cp[d], w_ih, w_hh, b_ih, b_hh, *w_hr)
                for got, want, S in ((hn[d], h64, S_h), (cn[d], c64, S_c)):
                    worst = max(worst, (np.abs(got - want)[live] / (KAPPA * u * S[live])).max(initial=0.0))
                assert (hn[d][~live] == hp[d][~live]).all() and (cn[d][~live] == cp[d][~live]).all(), (name, t)
            h, c = h1, c1
    _record_ratio("per_step_max_err_over_bound", name + ("_ragged" if ragged else ""), regime, "T%d" % T, worst)
    assert worst <= 1.0, (name, regime, ragged, worst)


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("ragged", [False, True], ids=["fixed", "ragged"])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_per_step_error_within_rounding_bound(name, ragged, regime):
    _per_step(name, regime, ragged, T=120 if regime == "saturated" else 40)


@pytest.mark.parametrize("name", ["gru256_tc8_3xtf32", "gru256_tc8_f16pair"])
def test_long_sequence_near_unit_spectral_radius(name, monkeypatch):
    """T = 500 with W_hh scaled to spectral radius ~1: state neither dies nor saturates, the per-step bound holds"""
    orig = _torch_model

    def model(*a, **k):
        ref = orig(*a, **k)
        with torch.no_grad():
            for n, p in ref.named_parameters():
                if n.startswith("weight_hh"):
                    rad = max(abs(np.linalg.eigvals(p[2 * p.shape[1]:].double().numpy())))
                    p.mul_(1.0 / rad)
        return ref

    monkeypatch.setattr(sys.modules[__name__], "_torch_model", model)
    _per_step(name, "default", False, T=500)


# ---- free running, calibrated against torch fp32 ----------------------------------------------------------------------

def _norm_err(a, ref64):
    a, ref64 = np.asarray(a, np.float64), np.asarray(ref64, np.float64)
    return np.linalg.norm(a - ref64) / max(np.linalg.norm(ref64), 1e-300)


def _run_torch(ref, x, lens, hx, wy, ws, dtype):
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

    m = ref.to(dtype)
    m.zero_grad()
    xx = x.to(dtype).clone().requires_grad_(True)
    st = [s.to(dtype).clone().requires_grad_(True) for s in hx]
    inp = xx if lens is None else pack_padded_sequence(xx, lens, enforce_sorted=False)
    out = m(inp, tuple(st) if len(st) == 2 else st[0])
    y = out[0] if lens is None else pad_packed_sequence(out[0], total_length=x.shape[0])[0]
    states = out[1] if isinstance(out[1], tuple) else (out[1],)
    loss = (y * wy.to(dtype)).sum() + sum((s * w.to(dtype)).sum() for s, w in zip(states, ws))
    loss.backward()
    res = {"y": y, **{k: s for k, s in zip(("h_n", "c_n"), states)}, "dx": xx.grad}
    res.update({"d" + n: p.grad for n, p in m.named_parameters()})
    res.update({k: s.grad for k, s in zip(("dh_0", "dc_0"), st)})
    return {k: v.detach().double().numpy() for k, v in res.items()}


def _run_mine(ref, mode, x, lens, hx, wy, ws):
    from b200rnn import from_torch
    from b200rnn.functional import rnn_forward

    mine = from_torch(ref.float()).to(DEV)
    xx = x.to(DEV).requires_grad_(True)
    st = [s.to(DEV).requires_grad_(True) for s in hx]
    out = rnn_forward(xx, mine._flat_weights, _cfg(mine, mode), lengths=lens, hx=tuple(st) if len(st) == 2 else st[0])
    y, states = out[0], out[1:]
    loss = (y * wy.to(DEV)).sum() + sum((s * w.to(DEV)).sum() for s, w in zip(states, ws))
    loss.backward()
    res = {"y": y, **{k: s for k, s in zip(("h_n", "c_n"), states)}, "dx": xx.grad}
    res.update({"d" + n: p.grad for n, p in mine.named_parameters()})
    res.update({k: s.grad for k, s in zip(("dh_0", "dc_0"), st)})
    return {k: v.detach().cpu().double().numpy() for k, v in res.items()}


@pytest.mark.parametrize("regime", ["default", "saturated", "large_input"])
@pytest.mark.parametrize("ragged", [False, True], ids=["fixed", "ragged"])
@pytest.mark.parametrize("name", [n for n in CONFIGS if CONFIGS[n][6] != "f16"])
def test_free_running_forward_backward_vs_f64(name, ragged, regime):
    kind, I, H, B, bi, P, mode = _shape(name, regime)
    T = 40
    ref = _torch_model(kind, I, H, bi, P, regime)
    x = _input(regime, T, B, I)
    lens = _ragged_lengths(B, T) if ragged else None
    if lens is not None:   # a row of length 0 keeps its initial state; torch packs only rows of length >= 1
        lens[1] = 1
    g = torch.Generator().manual_seed(4)
    D, HO = (2 if bi else 1), (P or H)
    hx = [0.5 * torch.randn(D, B, HO, generator=g)] + ([0.5 * torch.randn(D, B, H, generator=g)] if kind == "lstm" else [])
    wy = torch.randn(T, B, D * HO, generator=g)
    ws = [torch.randn(s.shape, generator=g) for s in hx]
    if lens is not None:
        wy = wy * (torch.arange(T)[:, None] < lens[None, :]).float()[:, :, None]
    r64 = _run_torch(ref, x, lens, hx, wy, ws, torch.float64)
    r32 = _run_torch(ref, x, lens, hx, wy, ws, torch.float32)
    mine = _run_mine(ref, mode, x, lens, hx, wy, ws)
    scale = 2.0 ** 13 if mode == "tf32" else 1.0
    bad = []
    for k, want in r64.items():
        e_k, e_t = _norm_err(mine[k], want), _norm_err(r32[k], want)
        _record_ratio("free_running_err_over_torch32", name + ("_ragged" if ragged else ""), regime, k,
                      e_k / max(e_t, 1e-300))
        if not e_k <= 4 * scale * e_t + 1e-6:
            bad.append((k, e_k, e_t))
    assert not bad, (name, regime, bad)


def test_f16_pair_forward_no_worse_than_3xtf32_saturated():
    """the no-grad fp16-pair forward keeps within 1.25 x the 3xTF32 module path's error in the saturated regime too"""
    from b200rnn import from_torch
    from oracle.rnn_numpy import NumpyRNN

    T, B = 120, 128
    ref = _torch_model("gru", 256, 256, False, 0, "saturated")
    mine = from_torch(ref).to(DEV)
    x = _input("saturated", T, B, 256)
    y16 = _forward(mine, "f16", x.to(DEV))[0].cpu().double().numpy()
    y32 = _forward(mine, "fp32", x.to(DEV))[0].cpu().double().numpy()
    y64 = NumpyRNN("gru", [p.detach().double().numpy() for p in ref.parameters()], 1, False).forward(
        x.double().numpy())[0]
    e16, e32 = np.abs(y16 - y64).max(), np.abs(y32 - y64).max()
    assert e16 <= 1.25 * e32 + 1e-6, (e16, e32)


# ---- every plan-table entry is reached ------------------------------------------------------------------------------

_CHILD = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}]
import torch
from b200rnn import from_torch
from b200rnn.functional import rnn_forward, rnn_forward_fused
torch.backends.cuda.matmul.fp32_precision = "ieee"
for name, (kind, I, H, B, bi, P, mode) in {configs!r}.items():
    for ragged in (False, True):
        if mode == "f16" and ragged:
            continue
        torch.manual_seed(0)
        cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
        m = from_torch(cls(I, H, bidirectional=bi, **({{"proj_size": P}} if P else {{}}))).to("cuda:0")
        cfg = m._config()
        cfg.tf32 = mode == "tf32"
        x = torch.randn(6, B, I, device="cuda:0", requires_grad=mode != "f16")
        lens = None
        if ragged:
            lens = torch.randint(1, 7, (B,))
            lens[0] = 6
        if mode == "f16":
            rnn_forward_fused(x, m._flat_weights, cfg)
        else:
            rnn_forward(x, m._flat_weights, cfg, lengths=lens)[0].sum().backward()
        torch.cuda.synchronize()
        print("[b200rnn] ran", name, int(ragged), file=sys.stderr, flush=True)
"""


def test_matrix_reaches_every_plan_table_entry():
    env = dict(os.environ, B200RNN_DEBUG="1")
    code = _CHILD.format(root=ROOT, pkg=PKG, configs=CONFIGS)
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    ran, fwd, bwd = {}, None, None
    for ln in proc.stderr.splitlines():
        if not ln.startswith("[b200rnn] "):
            continue
        body = ln[len("[b200rnn] "):]
        if body.startswith(("fwd cfg", "fwd proj cfg")):
            fwd = body.split(":")[0]
        elif body.startswith(("bwd cfg", "bwd proj cfg")):
            bwd = body.split(":")[0]
        elif body.startswith("ran "):
            _, name, ragged = body.split()
            ran[(name, ragged == "1")] = (fwd, bwd if CONFIGS[name][6] != "f16" else None)
            fwd = bwd = None
    want = {}
    for name in CONFIGS:
        for ragged in (False, True):
            if CONFIGS[name][6] == "f16" and ragged:
                continue
            want[(name, ragged)] = (FWD_LINE[name], BWD_LINE.get(name))
    assert ran == want, proc.stderr
    # every entry of both tables, each in its fixed-length and its ragged kernel (the f16 pair: fixed-length here)
    per_table = lambda i: {(CONFIGS[n][0], CONFIGS[n][2], v[i]) for (n, r), v in ran.items() if v[i]}  # noqa: E731
    assert len(per_table(0)) == N_FWD_ENTRIES and len(per_table(1)) == N_BWD_ENTRIES


# ---- non-finite padding and row isolation -----------------------------------------------------------------------------

def _module_run(ref, x, lens, wy, ws, hx):
    """forward + backward through rnn_forward(lengths=...): y, states, dx, parameter gradients, dh_0 / dc_0"""
    return _run_mine(ref, "fp32", x, lens, hx, wy, ws)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")], ids=["nan", "pinf", "ninf"])
@pytest.mark.parametrize("name", ["gru256_bs4", "gru256_tc8_3xtf32", "bilstm128", "bilstmp_h256_p64"])
def test_nonfinite_padding_reaches_nothing_module(name, bad):
    kind, I, H, B, bi, P, _ = CONFIGS[name]
    T = 24
    ref = _torch_model(kind, I, H, bi, P, "default")
    lens = _ragged_lengths(B, T)
    valid = (torch.arange(T)[:, None] < lens[None, :])[:, :, None]
    x = _input("default", T, B, I) * valid
    g = torch.Generator().manual_seed(9)
    D, HO = (2 if bi else 1), (P or H)
    hx = [0.5 * torch.randn(D, B, HO, generator=g)] + ([0.5 * torch.randn(D, B, H, generator=g)] if kind == "lstm" else [])
    wy = torch.randn(T, B, D * HO, generator=g)
    ws = [torch.randn(s.shape, generator=g) for s in hx]
    clean = _module_run(ref, x, lens, wy, ws, hx)
    dirty = _module_run(ref, torch.where(valid, x, torch.tensor(bad)), lens, wy, ws, hx)
    for k, v in clean.items():
        assert np.array_equal(dirty[k], v), (name, k)
    pad = ~valid.numpy()[:, :, 0]
    assert (dirty["y"][pad] == 0).all() and (dirty["dx"][pad] == 0).all()


def _abi_ln_fused(x_tm, lens, gru, ln_w, ln_b, dy):
    """b200rnn_forward_fused (SAVE_FOR_BACKWARD, LayerNorm prologue, lengths) and b200rnn_backward_fused with dy"""
    from b200rnn import _lib
    from b200rnn.functional import _make_desc, _stream_ptr

    lib = _lib.load()
    T, B, I = x_tm.shape
    H = gru.hidden_size
    desc = _make_desc(gru._config(), B, T, True, fused_ln=True)
    rbytes, sbytes = _lib.workspace_bytes(desc)
    reserve = torch.empty(rbytes, dtype=torch.uint8, device=DEV)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=DEV)
    y = torch.empty(T, B, H, device=DEV)
    h_n = torch.empty(1, B, H, device=DEV)
    params = _lib.ptr_array([w.data_ptr() for w in gru._flat_weights])
    ln32 = lens.to(DEV, torch.int32).contiguous()
    rc = lib.b200rnn_forward_fused(ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params,
                                   y.data_ptr(), B * H, H, h_n.data_ptr(), None, reserve.data_ptr(), scratch.data_ptr(),
                                   0, 0, None, ln_w.data_ptr(), ln_b.data_ptr(), 1e-5, None, ln32.data_ptr(), None,
                                   None, _stream_ptr(DEV))
    _lib.check(rc, "b200rnn_forward_fused")
    dx = torch.empty(T, B, I, device=DEV)
    grads = [torch.empty_like(w) for w in gru._flat_weights]
    dln_w, dln_b = torch.empty_like(ln_w), torch.empty_like(ln_b)
    dparams = _lib.ptr_array([g.data_ptr() for g in grads])
    rc = lib.b200rnn_backward_fused(ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params,
                                    y.data_ptr(), B * H, H, dy.data_ptr(), B * H, H, None, 0.0, None, None,
                                    reserve.data_ptr(), scratch.data_ptr(), dx.data_ptr(), B * I, I, dparams,
                                    ln32.data_ptr(), ln_w.data_ptr(), 1e-5, dln_w.data_ptr(), dln_b.data_ptr(),
                                    _stream_ptr(DEV))
    _lib.check(rc, "b200rnn_backward_fused")
    torch.cuda.synchronize()
    out = {"y": y, "h_n": h_n, "dx": dx, "dln_gamma": dln_w, "dln_beta": dln_b}
    out.update({"d%d" % i: g for i, g in enumerate(grads)})
    return {k: v.cpu() for k, v in out.items()}


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")], ids=["nan", "pinf", "ninf"])
def test_nonfinite_padding_reaches_nothing_abi_layernorm(bad):
    """the C ABI with the folded LayerNorm: the layer-0 dW_ih operand and the LayerNorm backward read the padded rows"""
    import b200rnn

    T, B, I, H = 24, 64, 256, 256
    torch.manual_seed(2)
    gru = b200rnn.GRU(I, H).to(DEV)
    g = torch.Generator().manual_seed(8)
    ln_w = (1 + 0.1 * torch.randn(I, generator=g)).to(DEV)
    ln_b = (0.1 * torch.randn(I, generator=g)).to(DEV)
    lens = _ragged_lengths(B, T)
    valid = (torch.arange(T)[:, None] < lens[None, :])[:, :, None]
    x = torch.randn(T, B, I, generator=g) * valid
    dy = (torch.randn(T, B, H, generator=g) * valid).to(DEV)
    clean = _abi_ln_fused(x.to(DEV), lens, gru, ln_w, ln_b, dy)
    dirty = _abi_ln_fused(torch.where(valid, x, torch.tensor(bad)).to(DEV), lens, gru, ln_w, ln_b, dy)
    for k, v in clean.items():
        assert torch.equal(dirty[k], v), k
    pad = ~valid[:, :, 0]
    assert (dirty["y"][pad] == 0).all() and (dirty["dx"][pad] == 0).all()


@pytest.mark.parametrize("name", list(CONFIGS))
def test_nan_in_one_row_stays_in_that_row(name):
    from b200rnn import from_torch

    kind, I, H, B, bi, P, mode = CONFIGS[name]
    T, t0, b0 = 16, 5, B // 2 + 1
    ref = _torch_model(kind, I, H, bi, P, "default")
    mine = from_torch(ref).to(DEV)
    x = _input("default", T, B, I)
    xp = x.clone()
    xp[t0, b0, I // 3] = float("nan")
    a = [o.cpu() for o in _forward(mine, mode, x.to(DEV))]
    p = [o.cpu() for o in _forward(mine, mode, xp.to(DEV))]
    others = torch.arange(B) != b0
    for u, v in zip(a, p):   # y [T,B,*], h_n / c_n [D,B,*]
        assert torch.equal(u[:, others], v[:, others]), name
    HO = P or H
    y = p[0][:, b0]
    assert torch.isnan(y[t0:, :HO]).all() and not torch.isnan(y[:t0, :HO]).any(), name
    if bi:   # the reverse half scans t = T-1 .. 0: poisoned at t0 and before
        assert torch.isnan(y[:t0 + 1, HO:]).all() and not torch.isnan(y[t0 + 1:, HO:]).any(), name
    for s in p[1:]:
        assert torch.isnan(s[:, b0]).all(), name
