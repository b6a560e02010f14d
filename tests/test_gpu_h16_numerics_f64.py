"""fp16 / bf16 GRU / LSTM / RNN modules against float64, off the easy path.

tests/test_gpu_h16_modules.py checks the 16-bit modules at torch's init with x ~ N(0, 1) and contiguous input. Here:

A. Route matrix. Every branch the 16-bit forward can take for its input projection (native wgmma reading x in place,
   native wgmma on a dense copy of x, the FFMA GEMM on widened copies; each direction's weight_ih on its own) and every
   recurrence config it reaches, each asserted from the B200RNN_DEBUG lines and the library's launch count, and each
   checked forward and backward against the float64 oracle of test_gpu_h16_modules.py in both dtypes.
B. Per step, teacher forced, rounding-exact. One-step calls chained through hx: the library widens the 16-bit state
   exactly, computes the step in fp32 and rounds once, so with v64 the float64 step from the same 16-bit operands
       |y16 - v64| <= ulp16(v64) / 2 + KAPPA u S        (KAPPA, u, S as in test_gpu_numerics_f64.py)
   and y16 == round16(v64) wherever v64 lies farther than KAPPA u S from a rounding midpoint (oracle/round16.py), which
   catches a double rounding, a truncation or a flush to zero. Applied to y, h_n and c_n.
C. Free running off default init: normwise per tensor, err_ours <= 4 err_cudnn + 1e-6, with err_cudnn stock torch in
   the same dtype on the GPU against the same oracle.
D. Edges: fp16 overflow to +-Inf exactly where float64 rounds there (outputs and gradients), subnormal outputs and
   subnormal inputs through both projection routes, non-finite padding of x and dy, NaN row isolation, and
   B200RNN_FLAG_ACCUMULATE_GRADS at the C ABI on the vector and the row path of the narrowing.
E. torch's fp32 matmul precision does not apply to 16-bit modules: "tf32" gives bitwise the "ieee" results.

B200RNN_NUMERICS_RECORD=<path> writes the per-case ratios (max err / bound, err_ours / err_cudnn) as JSON.
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import b200rnn
from oracle.rnn_numpy import elman_step, gru_step, lstm_step
from oracle.round16 import midpoint_distance, round16, ulp16
from test_gpu_h16_modules import MINE, STOCK, _kw, _oracle, _ulp
from test_gpu_numerics_f64 import BWD_LINE, FWD_LINE

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
KAPPA, U32 = 24.0, 2.0 ** -24
DT = {"f16": torch.float16, "bf16": torch.bfloat16}
REGIMES = ("default", "saturated", "large_input", "small_signal")
RECORDS = {}


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


# ---- models, inputs, checks ------------------------------------------------------------------------------------------

def _module(kind, I, H, dt, regime="default", bi=False, batch_first=False, seed=0):
    """a 16-bit module with the regime's weights (those of test_gpu_numerics_f64.py, then rounded to dt)"""
    torch.manual_seed(seed)
    mod = MINE[kind](I, H, bidirectional=bi, batch_first=batch_first, **_kw(kind))
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for n, p in mod.named_parameters():
            if regime == "saturated":
                if n.startswith("bias"):
                    p.copy_(torch.rand(p.shape, generator=g) * 6 - 3)
                    if kind == "lstm" and n.startswith("bias_ih"):
                        p[H:2 * H] += 3.0   # forget gate
                else:
                    p.mul_(4.0)
            elif regime == "small_signal" and n.startswith("bias"):
                p.mul_(1e-3)
    mod = mod.to(DEV, dt)
    mod._kind = kind
    return mod


def _input(regime, T, B, I, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, B, I, generator=g)
    return x * {"default": 1.0, "saturated": 2.0, "large_input": 30.0, "small_signal": 1e-3}[regime]


def _ragged_lengths(B, T, seed=3):
    lens = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(seed))
    lens[0], lens[1 % B], lens[2 % B] = T, 0, 1
    return lens


def _w64(mod, d=0):
    sfx = "_l0" + ("_reverse" if d else "")
    return [getattr(mod, n + sfx).detach().double().cpu().numpy() for n in ("weight_ih", "weight_hh", "bias_ih",
                                                                            "bias_hh")]


def _step64(kind, x, h, c, w):
    """float64 step from the 16-bit operands: (h', c' or None, S_h, S_c or None)"""
    if kind == "gru":
        h1, S = gru_step(x, h, *w)
        return h1, None, S, None
    if kind == "lstm":
        return lstm_step(x, h, c, *w)
    h1, S = elman_step(x, h, *w, nonlinearity=kind)
    return h1, None, S, None


def _rounded_once(got, v64, S, dt, what):
    """got (float64 copy of a 16-bit result) is v64 rounded once after an fp32 evaluation within KAPPA u S of it:
    equal to round16(v64) away from the midpoints, within half an ulp plus KAPPA u S everywhere. Returns the largest
    error over that bound (finite elements)."""
    e = KAPPA * U32 * S
    want = round16(v64, dt)
    exact = midpoint_distance(v64, dt) > e
    bad = exact & (got != want)
    assert not bad.any(), (what, got[bad][:4], want[bad][:4], v64[bad][:4])
    fin = np.isfinite(got) & np.isfinite(want)
    ratio = np.abs(got - v64)[fin] / (0.5 * ulp16(v64, dt)[fin] + e[fin])
    m = ratio.max(initial=0.0)
    assert m <= 1.0, (what, m)
    return m


def _np(t):
    return t.detach().double().cpu().numpy()


# ---- B. per step, teacher forced, rounding-exact --------------------------------------------------------------------

# one fixed-config H (GRU-256 and LSTM-128; the Elman RNN has only the runtime-sized kernels) and one runtime-sized H
PER_STEP = [("gru", 256), ("gru", 96), ("lstm", 128), ("lstm", 96), ("tanh", 256), ("tanh", 96), ("relu", 256),
            ("relu", 96)]


def _per_step(kind, H, dt, regime, ragged, T=8, B=16):
    from b200rnn.functional import rnn_forward

    I = 1024 if regime == "large_input" else 64
    mod = _module(kind, I, H, dt, regime)
    x = _input(regime, T, B, I).to(dt)
    x64 = x.double().numpy()
    w = _w64(mod)
    lens = _ragged_lengths(B, T) if ragged else None
    lstm = kind == "lstm"
    h = torch.zeros(1, B, H, dtype=dt, device=DEV)
    c = torch.zeros(1, B, H, dtype=dt, device=DEV) if lstm else None
    worst, steps = 0.0, 0
    for t in range(T):
        live = np.ones(B, bool) if lens is None else (t < lens.numpy())
        step_len = None if lens is None else torch.from_numpy(live.astype(np.int32))
        with torch.no_grad():
            out = rnn_forward(x[t:t + 1].to(DEV), mod._flat_weights, mod._config(), lengths=step_len,
                              hx=(h, c) if lstm else h)
        hp, cp = _np(h)[0], (_np(c)[0] if lstm else None)
        h64, c64, S_h, S_c = _step64(kind, x64[t], hp, cp, w)
        y1, h1 = _np(out[0])[0], _np(out[1])[0]
        checks = [(y1, h64, S_h, "y"), (h1, h64, S_h, "h_n")]
        if lstm:
            checks.append((_np(out[2])[0], c64, S_c, "c_n"))
        for got, want, S, what in checks:
            worst = max(worst, _rounded_once(got[live], want[live], S[live], dt, (kind, H, regime, t, what)))
        assert (y1[~live] == 0).all() and (h1[~live] == hp[~live]).all(), (kind, t)
        if lstm:
            assert (_np(out[2])[0][~live] == cp[~live]).all(), (kind, t)
        steps += 1
        if not np.isfinite(h1).all():   # fp16 relu grown past the range: the chain ends at the first Inf
            break
        h, c = out[1], (out[2] if lstm else None)
    assert steps >= 2
    return worst


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("ragged", [False, True], ids=["fixed", "ragged"])
@pytest.mark.parametrize("kind,H", PER_STEP)
@pytest.mark.parametrize("dtn", list(DT))
def test_per_step_rounded_once_from_float64(dtn, kind, H, ragged, regime):
    worst = _per_step(kind, H, DT[dtn], regime, ragged)
    _record_ratio("per_step_max_err_over_bound", f"{kind}{H}_{dtn}" + ("_ragged" if ragged else ""), regime, "T8",
                  worst)


# ---- C. free running, calibrated against cuDNN in the same dtype ----------------------------------------------------

def _norm_err(a, ref):
    return np.linalg.norm(a - ref) / max(np.linalg.norm(ref), 1e-300)


def _fwd_bwd(mod_or_stock, x, state, wy, ws, lstm):
    """forward + backward of a module on the GPU: {name: float64 array} of outputs and every gradient"""
    xx = x.to(DEV).requires_grad_(True)
    st = [s.to(DEV).requires_grad_(True) for s in state]
    for p in mod_or_stock.parameters():
        p.grad = None
    out = mod_or_stock(xx, tuple(st) if lstm else st[0])
    fin = list(out[1]) if lstm else [out[1]]
    loss = (out[0].float() * wy.to(DEV).float()).sum() + sum((f.float() * w.to(DEV).float()).sum()
                                                             for f, w in zip(fin, ws))
    loss.backward()
    res = {"y": out[0], "h_n": fin[0], "dx": xx.grad, "dh_0": st[0].grad}
    if lstm:
        res.update(c_n=fin[1], dc_0=st[1].grad)
    res.update({"d" + n: p.grad for n, p in mod_or_stock.named_parameters()})
    return {k: _np(v) for k, v in res.items()}


@pytest.mark.parametrize("regime", ["saturated", "large_input"])
@pytest.mark.parametrize("kind,H", [("gru", 256), ("gru", 96), ("lstm", 128), ("lstm", 640), ("tanh", 96)])
@pytest.mark.parametrize("dtn", list(DT))
def test_free_running_no_worse_than_cudnn(dtn, kind, H, regime):
    dt = DT[dtn]
    T, B = 40, 16
    I = 1024 if regime == "large_input" else 64
    lstm = kind == "lstm"
    mod = _module(kind, I, H, dt, regime)
    x = _input(regime, T, B, I).to(dt)
    g = torch.Generator().manual_seed(4)
    state = [(0.5 * torch.randn(1, B, H, generator=g)).to(dt) for _ in range(2 if lstm else 1)]
    wy = torch.randn(T, B, H, generator=g).to(dt)
    ws = [torch.randn(1, B, H, generator=g).to(dt) for _ in state]
    mine = _fwd_bwd(mod, x, state, wy, ws, lstm)
    stock = STOCK[kind](I, H, dtype=dt, **_kw(kind)).to(DEV)
    stock.load_state_dict(mod.state_dict())
    cudnn = _fwd_bwd(stock, x, state, wy, ws, lstm)
    ref, xin, h0, params = _oracle(mod, x.to(DEV), tuple(s.to(DEV) for s in state) if lstm else state[0].to(DEV), dt)
    ((ref[0] * wy.double()).sum() + sum((r * w.double()).sum() for r, w in zip(ref[1:], ws))).backward()
    want = {"y": ref[0], "h_n": ref[1], "dx": xin.grad, "dh_0": h0[0].grad}
    if lstm:
        want.update(c_n=ref[2], dc_0=h0[1].grad)
    want.update({"d" + n: p.grad for (n, _), p in zip(mod.named_parameters(), params)})
    bad = []
    for k, w64 in want.items():
        w64 = w64.detach().numpy()
        e_m, e_c = _norm_err(mine[k], w64), _norm_err(cudnn[k], w64)
        _record_ratio("free_running_err_over_cudnn", f"{kind}{H}_{dtn}", regime, k, e_m / max(e_c, 1e-300))
        if not e_m <= 4 * e_c + 1e-6:
            bad.append((k, e_m, e_c))
    assert not bad, (kind, H, dtn, regime, bad)


# ---- A. route matrix --------------------------------------------------------------------------------------------------

# name -> kind, I, H, B, layout, bidirectional, misaligned weight_ih directions, expectations
#   layout: "tm" contiguous time-major, "bf" batch_first, "colslice" x[..., :I] of a [T, B, I + 3] tensor (row stride
#   not 16-byte aligned), "offset1" x starting one element into its buffer
#   expectations: native = number of "weights=native" projection lines, copy = the copy16 launch of a dense copy
#   (batch 5 does not divide the 128-row tile, so the TMA cannot read those rows in place),
#   fwd / bwd = the recurrence config line (None: not asserted)
ROUTES = {
    "native_in_place": ("gru", 64, 128, 8, "tm", False, (), dict(native=1, copy=0)),
    "native_copy_batch_first_b5": ("gru", 64, 128, 5, "bf", False, (), dict(native=1, copy=1)),
    "native_copy_col_slice": ("lstm", 64, 128, 8, "colslice", False, (), dict(native=1, copy=1)),
    "native_copy_offset1": ("tanh", 64, 128, 8, "offset1", False, (), dict(native=1, copy=1)),
    "ffma_i33": ("gru", 33, 128, 8, "tm", False, (), dict(native=0, copy=0)),
    "ffma_i36": ("lstm", 36, 128, 8, "tm", False, (), dict(native=0, copy=0)),
    "ffma_gru48": ("gru", 64, 48, 8, "tm", False, (), dict(native=0, copy=0)),
    "ffma_w_ih_offset1": ("relu", 64, 128, 8, "tm", False, (0,), dict(native=0, copy=0)),
    "mixed_reverse_w_ih_offset1": ("gru", 64, 128, 8, "tm", True, (1,), dict(native=1, copy=0)),
    "gru256_bs2": ("gru", 256, 256, 16, "tm", False, (), dict(native=1, fwd=FWD_LINE["gru256_bs2"],
                                                             bwd=BWD_LINE["gru256_bs2"])),
    "gru256_bs4": ("gru", 256, 256, 64, "tm", False, (), dict(native=1, fwd=FWD_LINE["gru256_bs4"],
                                                             bwd=BWD_LINE["gru256_bs4"])),
    "gru256_tc8": ("gru", 256, 256, 128, "tm", False, (), dict(native=1, fwd=FWD_LINE["gru256_tc8_3xtf32"],
                                                              bwd=BWD_LINE["gru256_tc8_3xtf32"])),
    "gru128": ("gru", 40, 128, 64, "tm", False, (), dict(native=1, fwd=FWD_LINE["gru128"], bwd=BWD_LINE["gru128"])),
    "gru128_wide": ("gru", 40, 128, 272, "tm", False, (), dict(native=1, fwd=FWD_LINE["gru128_wide"],
                                                              bwd=BWD_LINE["gru128_wide"])),
    "bilstm128": ("lstm", 256, 128, 16, "tm", True, (), dict(native=2, fwd=FWD_LINE["bilstm128"],
                                                            bwd=BWD_LINE["bilstm128"])),
    "bilstm128_wide": ("lstm", 256, 128, 136, "tm", True, (), dict(native=2, fwd=FWD_LINE["bilstm128_wide"],
                                                                  bwd=BWD_LINE["bilstm128_wide"])),
    "bilstm256": ("lstm", 256, 256, 32, "tm", True, (), dict(native=2, fwd=FWD_LINE["bilstm256"],
                                                            bwd=BWD_LINE["bilstm256"])),
    "bilstm256_wide": ("lstm", 256, 256, 64, "tm", True, (), dict(native=2, fwd=FWD_LINE["bilstm256_wide"],
                                                                 bwd=BWD_LINE["bilstm256_wide"])),
    # the runtime-sized GRU forward keeps 16-bit W_hh on chip up to H = 752 (DESIGN.md, 16-bit modules); 3 * 752 is no
    # multiple of 128, so that projection runs on the FFMA GEMM
    "anyh_gru752_smem": ("gru", 64, 752, 8, "tm", False, (), dict(native=0, fwd="fwd anyh cfg GRU VL=0 H=752",
                                                                 fwd_tier="tier=smem w_hh=16bit")),
    "anyh_gru768_l2": ("gru", 64, 768, 8, "tm", False, (), dict(native=1, fwd="fwd anyh cfg GRU VL=0 H=768",
                                                               fwd_tier="tier=l2 w_hh=16bit")),
}
T_ROUTE = 6


def _route_inputs(name, dt, seed=0):
    """the case's module, its weights as passed to rnn_forward (misaligned copies where asked), x in the case's
    layout, a dense time-major x with the same values, and a dense time-major x of 8 rows, which the TMA reads in
    place (the launch count of the case minus that of this one is the dense copy's launch)"""
    kind, I, H, B, layout, bi, mis, _ = ROUTES[name]
    mod = _module(kind, I, H, dt, bi=bi, batch_first=layout == "bf", seed=seed)
    weights = list(mod._flat_weights)
    for d in mis:   # weight_ih of direction d, contiguous one element into a buffer
        w = weights[4 * d]
        buf = torch.zeros(w.numel() + 1, dtype=dt, device=DEV)
        buf[1:].copy_(w.flatten())
        weights[4 * d] = buf[1:].view_as(w).detach().requires_grad_(True)
        assert weights[4 * d].data_ptr() % 16 != 0
    g = torch.Generator().manual_seed(seed + 1)
    x_tm = torch.randn(T_ROUTE, B, I, generator=g).to(dt).to(DEV)
    if layout == "bf":
        x = x_tm.transpose(0, 1).contiguous()
        dense = x_tm.transpose(0, 1)   # a batch_first view of dense time-major rows
    elif layout == "colslice":
        wide = torch.zeros(T_ROUTE, B, I + 3, dtype=dt, device=DEV)
        wide[..., :I] = x_tm
        x, dense = wide[..., :I], x_tm
    elif layout == "offset1":
        buf = torch.zeros(x_tm.numel() + 1, dtype=dt, device=DEV)
        buf[1:].copy_(x_tm.flatten())
        x, dense = buf[1:].view_as(x_tm), x_tm
        assert x.data_ptr() % 16 != 0
    else:
        x, dense = x_tm, x_tm
    ref = torch.randn(T_ROUTE, 8, I, generator=g).to(dt).to(DEV)
    return mod, weights, x, dense, (ref.transpose(0, 1) if layout == "bf" else ref)


_ROUTE_CHILD = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}, {tests!r}]
import torch
from b200rnn import _lib
from b200rnn.functional import rnn_forward
import test_gpu_h16_numerics_f64 as t
torch.backends.cuda.matmul.fp32_precision = {precision!r}
for dtn in ("f16", "bf16"):
    for name in t.ROUTES:
        mod, weights, x, dense, ref = t._route_inputs(name, t.DT[dtn])
        cfg = mod._config()
        with torch.no_grad():
            rnn_forward(ref, weights, cfg)
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            rnn_forward(ref, weights, cfg)
            torch.cuda.synchronize()
            n1 = _lib.launch_count()
        print("[b200rnn] case", dtn, name, file=sys.stderr, flush=True)
        with torch.no_grad():
            rnn_forward(x, weights, cfg)
            torch.cuda.synchronize()
        n2 = _lib.launch_count()
        rnn_forward(x.detach().requires_grad_(True), weights, cfg)[0].float().sum().backward()
        torch.cuda.synchronize()
        print("[b200rnn] ran", dtn, name, (n2 - n1) - (n1 - n0), file=sys.stderr, flush=True)
"""


def _route_lines(precision):
    code = _ROUTE_CHILD.format(root=ROOT, pkg=PKG, tests=os.path.join(ROOT, "tests"), precision=precision)
    env = dict(os.environ, B200RNN_DEBUG="1")
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout + proc.stderr[-4000:]
    cases, cur = {}, None
    for ln in proc.stderr.splitlines():
        if not ln.startswith("[b200rnn] "):
            continue
        body = ln[len("[b200rnn] "):]
        if body.startswith("case "):
            cur = tuple(body.split()[1:3])
            cases[cur] = {"lines": []}
        elif body.startswith("ran "):
            _, dtn, name, extra = body.split()
            cases[(dtn, name)]["copy"] = int(extra)
            cur = None
        elif cur is not None:
            cases[cur]["lines"].append(body)
    return cases


def _assert_routes(cases, dtn, name):
    kind, I, H, B, layout, bi, mis, want = ROUTES[name]
    got = cases[(dtn, name)]
    lines = got["lines"]
    fwd_lines = [ln for ln in lines if ln.startswith("forward x-projection")]
    native = [ln for ln in fwd_lines if "weights=native" in ln]
    # the lines of the first (no-grad) forward and of the forward under autograd: each projection twice
    assert len(native) == 2 * want["native"], (dtn, name, lines)
    assert all(f"math={dtn} weights=native" in ln for ln in native), (dtn, name, native)
    assert all("weights=native" in ln for ln in fwd_lines), (dtn, name, fwd_lines)   # no TF32 / 3xTF32 GEMM on x
    if "copy" in want:
        assert got["copy"] == want["copy"], (dtn, name, got["copy"])
    if "fwd" in want:
        assert any(ln.startswith(want["fwd"]) and want.get("fwd_tier", "") in ln for ln in lines), (dtn, name, lines)
    if "bwd" in want:
        assert any(ln.startswith(want["bwd"]) for ln in lines), (dtn, name, lines)


def test_route_matrix_reaches_every_16bit_branch():
    """the B200RNN_DEBUG lines and launch counts of every case, in default precision"""
    cases = _route_lines("ieee")
    assert set(cases) == {(d, n) for d in DT for n in ROUTES}
    for dtn in DT:
        for name in ROUTES:
            _assert_routes(cases, dtn, name)


def test_tf32_setting_leaves_16bit_routes_alone():
    """torch's fp32 matmul precision "tf32" changes no 16-bit route: GRU-256 at B = 128 stays 3xTF32 on tc8"""
    cases = _route_lines("tf32")
    for dtn in DT:
        for name in ROUTES:
            _assert_routes(cases, dtn, name)
        assert not any("TF32" in ln and "3xTF32" not in ln for ln in cases[(dtn, "gru256_tc8")]["lines"])


@pytest.mark.parametrize("name", list(ROUTES))
@pytest.mark.parametrize("dtn", list(DT))
def test_route_matrix_against_float64(dtn, name):
    """each route, forward and every gradient against the float64 oracle with test_gpu_h16_modules.py's bounds"""
    from b200rnn.functional import rnn_forward

    dt = DT[dtn]
    kind, I, H, B, layout, bi, mis, _ = ROUTES[name]
    mod, weights, x, dense, _ = _route_inputs(name, dt)
    xx = x.detach().requires_grad_(True)
    for w in weights:
        w.grad = None
    out = rnn_forward(xx, weights, mod._config())
    finals = list(out[1:])
    g = torch.Generator().manual_seed(7)
    wy = torch.randn(out[0].shape, generator=g).to(dt).to(DEV)
    ((out[0].float() * wy.float()).sum() + sum(f.float().sum() for f in finals)).backward()
    ref, xin, _, params = _oracle(mod, dense, None, dt)
    ((ref[0] * wy.double().cpu()).sum() + sum(r.sum() for r in ref[1:])).backward()
    for got, want in zip([out[0]] + finals, ref):
        gg, r = got.double().cpu(), want.detach()
        bound = torch.tensor([0.5 * _ulp(v, dt) for v in r.flatten().tolist()]).view_as(r) + 2e-5
        assert ((gg - r).abs() <= bound).all(), (name, dtn, (gg - r).abs().max().item())
    for got, want in [(xx.grad, xin.grad)] + [(w.grad, q.grad) for w, q in zip(weights, params)]:
        assert got is not None and got.dtype == dt
        m = want.abs().max().item()
        err = (got.double().cpu() - want).abs().max().item()
        assert err <= _ulp(m, dt) + 1e-4 * m, (name, dtn, err, m)


# ---- D. edges ---------------------------------------------------------------------------------------------------------

def _relu_layer(I, H, dt, B, w_ih_scale, seed=0, x=None, zero_bias=False, hx=True):
    """one relu step (T = 1) with weight_ih scaled, forward and backward of loss = sum(y * dy); returns the module,
    its tensors and the results"""
    mod = _module("relu", I, H, dt, seed=seed)
    with torch.no_grad():
        mod.weight_ih_l0.mul_(w_ih_scale)
        if zero_bias:
            mod.bias_ih_l0.zero_()
            mod.bias_hh_l0.zero_()
    g = torch.Generator().manual_seed(seed + 1)
    if x is None:
        x = torch.randn(1, B, I, generator=g).to(dt)
    x = x.to(DEV).requires_grad_(True)
    h0 = (0.5 * torch.randn(1, B, H, generator=g)).to(dt).to(DEV).requires_grad_(True) if hx else None
    dy = torch.randn(1, B, H, generator=g).to(dt).to(DEV)
    y, _ = mod(x, h0)
    y.backward(dy)
    return mod, x, h0, dy, y


@pytest.mark.parametrize("dtn", list(DT))
def test_overflow_is_inf_exactly_where_float64_rounds_there(dtn):
    """relu RNN with |y| and |dx| around 65520: fp16 gives +-Inf exactly where the float64 value rounds to it and is
    correctly rounded elsewhere; bf16 stays finite"""
    dt = DT[dtn]
    I, H, B = 64, 128, 64
    mod, x, h0, dy, y = _relu_layer(I, H, dt, B, 1e5)
    w = _w64(mod)
    x64, h64 = _np(x)[0], _np(h0)[0]
    v64, S = elman_step(x64, h64, *w, nonlinearity="relu")
    y16 = _np(y)[0]
    _rounded_once(y16, v64, S, dt, "y")
    pre = x64 @ w[0].T + w[2] + h64 @ w[1].T + w[3]
    dpre = _np(dy)[0] * (pre > 0)
    dx64, S_dx = dpre @ w[0], np.abs(dpre) @ np.abs(w[0])
    _rounded_once(_np(x.grad)[0], dx64, S_dx, dt, "dx")
    if dt == torch.float16:
        assert np.isinf(y16).sum() >= 20 and (np.isfinite(y16) & (y16 > 30000)).sum() >= 20
        gx = _np(x.grad)[0]
        assert (gx == np.inf).sum() >= 20 and (gx == -np.inf).sum() >= 20 and (np.abs(gx[np.isfinite(gx)]) > 30000).any()
    else:
        assert np.isfinite(y16).all() and np.isfinite(_np(x.grad)).all() and y16.max() > 65520


def test_fp16_subnormal_outputs_are_rounded_not_flushed():
    """small_signal scaled further: relu outputs in fp16's subnormal range, each correctly rounded"""
    dt = torch.float16
    I, H, B = 64, 128, 64
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(1, B, I, generator=g) * 1e-2).to(dt)
    mod, x, _, _, y = _relu_layer(I, H, dt, B, 1e-3, x=x, zero_bias=True, hx=False)
    w = _w64(mod)
    v64, S = elman_step(_np(x)[0], np.zeros((B, H)), *w, nonlinearity="relu")
    y16 = _np(y)[0]
    _rounded_once(y16, v64, S, dt, "y")
    sub = (y16 > 0) & (y16 < 2.0 ** -14)
    assert sub.sum() >= B * H // 8, sub.sum()


@pytest.mark.parametrize("I", [64, 36], ids=["native", "ffma"])
@pytest.mark.parametrize("dtn", list(DT))
def test_subnormal_input_products_are_exact(dtn, I):
    """x subnormal in the dtype (fp16 k 2^-24; bf16 k 2^-133) against weight_ih of 2^10 / 2^100: every product is
    exact in fp32 and normal, so the output is the correctly rounded sum, on wgmma and on the FFMA GEMM"""
    dt = DT[dtn]
    H, B = 128, 64
    g = torch.Generator().manual_seed(6)
    k = torch.randint(-1023 if dt == torch.float16 else -127, 1024 if dt == torch.float16 else 128, (1, B, I),
                      generator=g).double()
    x = (k * 2.0 ** (-24 if dt == torch.float16 else -133)).to(dt)
    assert (x.double() == k * 2.0 ** (-24 if dt == torch.float16 else -133)).all()
    scale = 2.0 ** 10 if dt == torch.float16 else 2.0 ** 100
    mod, x, _, _, y = _relu_layer(I, H, dt, B, scale * (H ** 0.5), x=x, zero_bias=True, hx=False)
    w = _w64(mod)
    v64, S = elman_step(_np(x)[0], np.zeros((B, H)), *w, nonlinearity="relu")
    y16 = _np(y)[0]
    _rounded_once(y16, v64, S, dt, "y")
    assert (y16 > 0).sum() >= B * H // 4


def _masked_run(mod, weights, x, lens, dy, dh, h0):
    from b200rnn.functional import rnn_forward

    xx = x.detach().clone().requires_grad_(True)
    hh = h0.detach().clone().requires_grad_(True)
    ws = [w.detach().clone().requires_grad_(True) for w in weights]
    y, h_n = rnn_forward(xx, ws, mod._config(), lengths=lens, hx=hh)
    torch.autograd.backward([y, h_n], [dy, dh])
    out = {"y": y, "h_n": h_n, "dx": xx.grad, "dh_0": hh.grad}
    out.update({"d%d" % i: w.grad for i, w in enumerate(ws)})
    return {k: v.detach().cpu() for k, v in out.items()}


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")], ids=["nan", "pinf", "ninf"])
@pytest.mark.parametrize("I", [64, 36], ids=["native", "ffma"])
@pytest.mark.parametrize("dtn", list(DT))
def test_nonfinite_padding_reaches_nothing(dtn, I, bad):
    """NaN / +-Inf in the padded rows of x and of dy: outputs and every gradient bitwise those of the clean run, padded
    y and dx rows 0 (the backward widens all of x and keeps 0 * NaN out of dW_ih by zeroing the padding)"""
    dt = DT[dtn]
    T, B, H = 12, 8, 128
    mod = _module("gru", I, H, dt, bi=True)
    lens = _ragged_lengths(B, T)
    valid = (torch.arange(T)[:, None] < lens[None, :])[:, :, None].to(DEV)
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(T, B, I, generator=g).to(dt).to(DEV)) * valid
    dy = torch.randn(T, B, 2 * H, generator=g).to(dt).to(DEV) * valid
    dh = torch.randn(2, B, H, generator=g).to(dt).to(DEV)
    h0 = (0.5 * torch.randn(2, B, H, generator=g)).to(dt).to(DEV)
    fill = torch.tensor(bad, dtype=dt, device=DEV)
    clean = _masked_run(mod, mod._flat_weights, x, lens, dy, dh, h0)
    dirty = _masked_run(mod, mod._flat_weights, torch.where(valid, x, fill), lens, torch.where(valid, dy, fill), dh, h0)
    for k, v in clean.items():
        assert torch.equal(dirty[k], v), (k, dtn, I)
    pad = ~valid[:, :, 0].cpu()
    assert (dirty["y"][pad] == 0).all() and (dirty["dx"][pad] == 0).all()


@pytest.mark.parametrize("I", [64, 36], ids=["native", "ffma"])
@pytest.mark.parametrize("dtn", list(DT))
def test_nan_in_one_row_stays_in_that_row(dtn, I):
    dt = DT[dtn]
    T, B, H, t0, b0 = 12, 8, 128, 5, 3
    mod = _module("gru", I, H, dt, bi=True)
    x = torch.randn(T, B, I, generator=torch.Generator().manual_seed(2)).to(dt).to(DEV)
    xp = x.clone()
    xp[t0, b0, I // 3] = float("nan")
    with torch.no_grad():
        a = [o.cpu() for o in mod(x)]
        p = [o.cpu() for o in mod(xp)]
    others = torch.arange(B) != b0
    assert torch.equal(a[0][:, others], p[0][:, others]) and torch.equal(a[1][:, others], p[1][:, others])
    y = p[0][:, b0]
    assert torch.isnan(y[t0:, :H]).all() and not torch.isnan(y[:t0, :H]).any()
    assert torch.isnan(y[:t0 + 1, H:]).all() and not torch.isnan(y[t0 + 1:, H:]).any()
    assert torch.isnan(p[1][:, b0]).all()


def _abi_accumulate(mod, x, h0, dy, targets):
    """b200rnn_forward_hx (SAVE_FOR_BACKWARD) then b200rnn_backward_hx with ACCUMULATE_GRADS into `targets`"""
    from b200rnn import _lib
    from b200rnn.functional import _make_desc, _stream_ptr

    lib = _lib.load()
    T, B, I = x.shape
    H = mod.hidden_size
    cfg = mod._config()
    desc = _make_desc(cfg, B, T, True)
    rbytes, sbytes = _lib.workspace_bytes(desc)
    reserve = torch.empty(rbytes, dtype=torch.uint8, device=DEV)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=DEV)
    y = torch.empty(T, B, H, dtype=x.dtype, device=DEV)
    h_n = torch.empty(1, B, H, dtype=x.dtype, device=DEV)
    params = _lib.ptr_array([w.data_ptr() for w in mod._flat_weights])
    _lib.check(lib.b200rnn_forward_hx(ctypes.byref(desc), x.data_ptr(), x.stride(0), x.stride(1), params, y.data_ptr(),
                                      B * H, H, h0.data_ptr(), None, h_n.data_ptr(), None, reserve.data_ptr(),
                                      scratch.data_ptr(), 0, 0, None, None, _stream_ptr(DEV)), "forward_hx")
    dacc = _make_desc(cfg, B, T, True, accumulate=True)
    _, sbytes = _lib.workspace_bytes(dacc)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=DEV)
    dx = torch.empty_like(x)
    dh0 = torch.empty_like(h0)
    dparams = _lib.ptr_array([t.data_ptr() for t in targets])
    _lib.check(lib.b200rnn_backward_hx(ctypes.byref(dacc), x.data_ptr(), x.stride(0), x.stride(1), params, y.data_ptr(),
                                       B * H, H, dy.data_ptr(), B * H, H, None, None, h0.data_ptr(), None,
                                       dh0.data_ptr(), None, reserve.data_ptr(), scratch.data_ptr(), dx.data_ptr(),
                                       B * I, I, dparams, None, _stream_ptr(DEV)), "backward_hx")
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize("path", ["vector", "row"])
@pytest.mark.parametrize("dtn", list(DT))
def test_accumulate_grads_rounds_once(dtn, path):
    """B200RNN_FLAG_ACCUMULATE_GRADS: each 16-bit gradient becomes one rounding of old + g (the fp32 gradient added to
    the widened old value), on the vector path of the narrowing and on its row path (I = 33, targets one element
    into their buffers)"""
    dt = DT[dtn]
    I, H, B = (64, 128, 32) if path == "vector" else (33, 128, 32)
    mod = _module("relu", I, H, dt)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, B, I, generator=g).to(dt).to(DEV)
    h0 = (0.5 * torch.randn(1, B, H, generator=g)).to(dt).to(DEV)
    dy = torch.randn(1, B, H, generator=g).to(dt).to(DEV)
    olds, targets = [], []
    for w in mod._flat_weights:
        old = (torch.randn(w.shape, generator=g) * 4).to(dt).to(DEV)
        if path == "row":
            buf = torch.zeros(w.numel() + 1, dtype=dt, device=DEV)
            t = buf[1:].view_as(w)
            assert t.data_ptr() % 8 != 0
        else:
            t = torch.empty_like(w)
        t.copy_(old)
        olds.append(_np(old))
        targets.append(t)
    _abi_accumulate(mod, x, h0, dy, targets)
    w = _w64(mod)
    x64, h64, dy64 = _np(x)[0], _np(h0)[0], _np(dy)[0]
    pre = x64 @ w[0].T + w[2] + h64 @ w[1].T + w[3]
    dpre = dy64 * (pre > 0)
    grads = [(dpre.T @ x64, np.abs(dpre).T @ np.abs(x64)), (dpre.T @ h64, np.abs(dpre).T @ np.abs(h64)),
             (dpre.sum(0), np.abs(dpre).sum(0)), (dpre.sum(0), np.abs(dpre).sum(0))]
    for i, ((g64, S), old, t) in enumerate(zip(grads, olds, targets)):
        _rounded_once(_np(t), old + g64, S + np.abs(old), dt, ("accumulate", i))


# ---- E. TF32 mode -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,H,B,I", [("gru", 256, 128, 256), ("lstm", 640, 16, 64)])
@pytest.mark.parametrize("dtn", list(DT))
def test_tf32_setting_does_not_change_16bit_results(dtn, kind, H, B, I):
    """16-bit modules do not follow torch's fp32 matmul precision (cuDNN's 16-bit RNNs do not either): forward and
    every gradient under "tf32" are bitwise those under "ieee" (GRU-256 at B = 128 runs tc8 on its fp32 W_hh copy)"""
    dt = DT[dtn]
    T = 10
    lstm = kind == "lstm"
    mod = _module(kind, I, H, dt)
    x = _input("default", T, B, I).to(dt)
    g = torch.Generator().manual_seed(4)
    state = [(0.5 * torch.randn(1, B, H, generator=g)).to(dt) for _ in range(2 if lstm else 1)]
    wy = torch.randn(T, B, H, generator=g).to(dt)
    ws = [torch.randn(1, B, H, generator=g).to(dt) for _ in state]
    prev = torch.backends.cuda.matmul.fp32_precision
    try:
        torch.backends.cuda.matmul.fp32_precision = "ieee"
        a = _fwd_bwd(mod, x, state, wy, ws, lstm)
        torch.backends.cuda.matmul.fp32_precision = "tf32"
        assert b200rnn.functional.tf32_enabled()
        b = _fwd_bwd(mod, x, state, wy, ws, lstm)
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), (k, np.abs(a[k] - b[k]).max())
