"""Forward-mode AD (b200rnn_forward_tangent, anyh_tangent_kernel, the linearised cells of csrc/rnn_cell.cuh) against
float64, away from default init.

test_gpu_jvp.py checks each tangent within 1e-4 of the tensor's largest entry, which cannot tell an fp32-accurate tangent
from a TF32-accurate one and hides any error in the small entries. Here the tangent answers to the bounds the other
float64 suites use (test_gpu_numerics_f64.py, test_gpu_anyh_numerics_f64.py), in the regimes default, saturated (radius
for the relu RNN), large_input and small_signal of those suites, with N(0, 1) tangents in every input.

Per-step test (teacher forced). Each step of the kernel's own tangent trajectory is recomputed in float64 from the
kernel's previous primal and tangent state (oracle.rnn_numpy.gru_step_jvp / lstm_step_jvp / elman_step_jvp), and every
element must satisfy

    |h'_kernel - step_jvp64(h_prev_kernel, h'_prev_kernel)| <= KAPPA_T * u * S'

with u = 2^-24 and S' the oracle's magnitude: the rounding of the tangent's own terms plus the primal's error (the kernel
applies the linearised cell at its saved activations, within KAPPA u S of float64) times the tangent magnitudes that
error scales (rnn_numpy.py). KAPPA_T counts rounding stages, as KAPPA does in test_gpu_numerics_f64.py:
  - each tangent pre-activation is one sum of at most 2 I + 2 H + 2 terms (W_ih x', W_ih' x, W_hh' h_{t-1}, W_hh h'_{t-1},
    b_ih', b_hh'), reached by at most 8 roundings at the sum's own magnitude: the stores of up to four GEMMs into the
    pre-activation buffer (the writing W_ih x', the accumulating W_ih' x, the row-shifted W_hh' h_{t-1} and the h_0 GEMM
    of the first step), the two bias tangents, the recurrent contraction's add and the combine; plus the error of the
    accumulations themselves. The FFMA GEMM and the recurrent contraction are serial FMA chains of up to K = 1024 (the
    large_input I, the largest H), sqrt(1024) = 32 (Higham & Mary, as in test_gpu_numerics_f64.py): 40 stages;
  - the linearised cell multiplies each pre-activation tangent by up to three saved factors (GRU r (1 - r) hn (1 - z)
    (1 - n^2) is the longest product) and adds up to four products: 8 stages, each against a term S' holds;
  - the primal's error enters through KAPPA = 24 <= KAPPA_T, which S' already carries as S Q.
KAPPA_T = 40 + 8 = 48. The kernels sit far inside it (tools/jvp_numerics_f64_results.json: below 0.1 of it). For the GRU
and LSTM the primal's share S Q dominates S', so this bound does not tell a TF32-accurate tangent from an fp32-accurate
one (tests/test_jvp_oracle_cpu.py: a TF32-rounded fp32 evaluation stays inside it there, and exceeds it for the Elman
cell); what it catches is a wrong term of the linearised step. Precision is the free-running test's job.

GRU / Elman: one jvp call with tangents on every input; the previous primal state of row b at step t is the kernel's
y[t - 1] (reverse half: y[t + 1]) or h_0, its previous tangent the kernel's y'[t - 1] (y'[t + 1]) or h_0' - the rows of
the row-shifted W_hh' h_{t-1} GEMM and the reverse half's first-row offset. LSTM: chained one-step calls through (h, c)
and (h', c'), as in the primal's per-step tests. relu: the bound needs the kernel and float64 to take the same branch
at every element (y > 0 agrees), which is asserted (test_gpu_anyh_numerics_f64.py). small_signal is recorded, not
asserted: tanh_f errs by ~1e-7 absolute by design.

Shapes (STEP): GRU, LSTM, RNN tanh, RNN relu, both directions, with hx, in both weight tiers of the tangent kernel (which
plans its shape and tier as the runtime-sized forward does): on chip at H = 48, 96, 272 (uneven H / 8 groups) and 464 for
the relu RNN; in L2 at H = 464 (LSTM), 1008, 1024.

Free-running test. y', h_n' and c_n' of 1 - 3 layer modules, normwise per tensor, against float64 stock torch.func.jvp on
the CPU, with the bound of the other suites:

    err_kernel <= 4 * err_torch32 + 1e-6        (TF32 mode: err_torch32 scaled by 2^13)

err_torch32 is stock fp32 jvp on the CPU on the same inputs (the LSTM with mkldnn off: mkldnn_rnn_layer has no forward-AD
formula). In fp32 mode a tangent GEMM or exchange at TF32 precision fails it by orders of magnitude.

Every primal config. The tangent kernel reads the saving forward's reserve (gates, GRU W_hn h + b_hn, LSTM c_t), which at
H = 128 / 256 the fixed configs of plan_rec_fwd write: one free-running case per saving fp32 config of
test_gpu_numerics_f64.CONFIGS - gru256 bs2, bs4, tc8 3xTF32, tc8 TF32 (TF32 mode), gru128 / _wide, bilstm256 / _wide,
bilstm128 / _wide. Not reachable by a saving forward, so not here: the fp16-pair configs (gru256_tc8_f16pair,
bilstm128_tcl8_f16pair), which serve the no-grad fused forward only, and the projected bilstmp_* configs, whose forward
mode is refused (proj_size). A B200RNN_DEBUG child process shows each case's `fwd cfg` line and its tangent launch, each
per-step shape's tier, and that the batched cases' tangent launch shape does not depend on M.

Batched tangents (M > 1, vmap over jvp): each of x, W_ih', W_hh', the bias tangents alone (no W_hh', so b_hn' reaches the
GRU's h side through the kernel only), h_0', c_0', and all together, on chip and in L2, both directions, and M = 64 at
B = 200 (more clusters than one wave): each direction bitwise equal to the single-direction jvp of the same tangent. Train
mode with inter-layer dropout at M > 1: every direction against float64 with the primal's Philox masks.

Edges: T = 1 (no row-shifted GEMM, only the h_0 GEMM), B = 1, unbatched input; and the B == 0 / T == 0 early return of
b200rnn_forward_tangent with M = 3: h_n' / c_n' equal h_0' / c_0' per direction, and are zero without them.

B200RNN_NUMERICS_RECORD=<path> writes this file's ratios to jvp_numerics_f64_results.json beside <path>."""
import copy
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch.func import functional_call, jvp

from test_gpu_anyh_numerics_f64 import CONFIGS as ANYH_CONFIGS
from test_gpu_anyh_numerics_f64 import _hx, _tf32
from test_gpu_numerics_f64 import CONFIGS as FIXED_CONFIGS
from test_gpu_numerics_f64 import FWD_LINE, KAPPA, U32, _input, _norm_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
KAPPA_T = 48.0
assert KAPPA <= KAPPA_T
RECORDS = {}
MODE_NAME = {"gru": "GRU", "lstm": "LSTM", "rnn_tanh": "RNN_TANH", "rnn_relu": "RNN_RELU"}
REGIMES = ("default", "stress", "large_input", "small_signal")

# per-step shapes: name -> kind, I, H, B, bidirectional, the tangent kernel's weight tier on an H100
STEP = {**{n: c for n, c in ANYH_CONFIGS.items()},
        "gru_h48_bi": ("gru", 40, 48, 24, True, "smem"),
        "gru_h1024_bi": ("gru", 48, 1024, 6, True, "l2"),
        "lstm_h1024_bi": ("lstm", 48, 1024, 3, True, "l2")}
# free running: name -> kind, I, H, L, bidirectional, B, T, regime
FREE = {
    "gru_h272_L2_bi": ("gru", 64, 272, 2, True, 16, 40, "saturated"),
    "gru_h1024": ("gru", 48, 1024, 1, False, 6, 40, "default"),
    "gru_h48_L3_bi": ("gru", 1024, 48, 3, True, 12, 30, "large_input"),
    "lstm_h96_L3_bi": ("lstm", 40, 96, 3, True, 12, 40, "saturated"),
    "lstm_h464_bi": ("lstm", 1024, 464, 1, True, 8, 30, "large_input"),
    "tanh_h272_L2": ("rnn_tanh", 40, 272, 2, False, 16, 40, "saturated"),
    "tanh_h1008_bi": ("rnn_tanh", 1024, 1008, 1, True, 8, 30, "large_input"),
    "relu_h464_L2_bi": ("rnn_relu", 64, 464, 2, True, 16, 60, "radius"),
    "relu_h1024": ("rnn_relu", 48, 1024, 1, False, 6, 40, "default"),
}
# the saving fp32 forward configs of plan_rec_fwd (test_gpu_numerics_f64.CONFIGS without the fp16-pair and proj_size)
PRIMAL = [n for n, c in FIXED_CONFIGS.items() if c[6] != "f16" and not c[5]]
# batched tangents: name -> kind, I, H, L, bidirectional, B, M, tier
BATCH = {
    "gru_h48_L2_bi": ("gru", 24, 48, 2, True, 7, 5, "smem"),
    "lstm_h96_bi": ("lstm", 24, 96, 1, True, 7, 5, "smem"),
    "tanh_h272": ("rnn_tanh", 24, 272, 1, False, 5, 5, "smem"),
    "gru_h1024_bi": ("gru", 24, 1024, 1, True, 3, 4, "l2"),
    "lstm_h464_bi": ("lstm", 24, 464, 1, True, 4, 4, "l2"),
    "relu_h1024": ("rnn_relu", 24, 1024, 1, False, 3, 4, "l2"),
}
WAVE = ("gru", 24, 256, 1, True, 200, 64, "smem")   # M = 64 at B = 200: more clusters than one wave
BATCH_GROUPS = ("x", "weight_ih", "weight_hh", "bias", "h_0", "c_0", "all")


@pytest.fixture(scope="module", autouse=True)
def _record():
    yield
    path = os.environ.get("B200RNN_NUMERICS_RECORD")
    if path and RECORDS:
        with open(os.path.join(os.path.dirname(os.path.abspath(path)), "jvp_numerics_f64_results.json"), "w") as f:
            json.dump(RECORDS, f, indent=1, sort_keys=True)
            f.write("\n")


def _record_ratio(kind, name, regime, key, value):
    RECORDS.setdefault(kind, {}).setdefault(name, {}).setdefault(regime, {})[key] = float(value)


# ---- models, inputs and tangents --------------------------------------------------------------------------------------

def _stock(kind, I, H, L, bi, regime, seed=0, dropout=0.0):
    """stock torch module (fp32, CPU) with the regime's weights (test_gpu_anyh_numerics_f64._torch_model, any depth)"""
    torch.manual_seed(seed)
    if kind in ("gru", "lstm"):
        ref = (torch.nn.GRU if kind == "gru" else torch.nn.LSTM)(I, H, num_layers=L, bidirectional=bi, dropout=dropout)
    else:
        ref = torch.nn.RNN(I, H, num_layers=L, nonlinearity=kind[4:], bidirectional=bi, dropout=dropout)
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
            elif regime == "radius" and n.startswith("weight_hh"):
                p.mul_(0.95 / max(abs(np.linalg.eigvals(p.double().numpy()))))
    return ref


def _regime(kind, regime):
    return ("radius" if kind == "rnn_relu" else "saturated") if regime == "stress" else regime


def _inputs(kind, I, H, L, D, B, T, regime, unbatched=False):
    """x [T,B,I], hx ((h_0, c_0),) or (h_0,) and N(0, 1) tangents of x, hx and every parameter of `ref`"""
    x = _input("default" if regime == "radius" else regime, T, B, I)
    hx = _hx(kind, L * D, B, H)
    if unbatched:
        x, hx = x[:, 0], [h[:, 0] for h in hx]
    g = torch.Generator().manual_seed(7)
    rnd = lambda t: torch.randn(t.shape, generator=g)  # noqa: E731
    return x, (tuple(hx),) if kind == "lstm" else (hx[0],), rnd(x), (tuple(rnd(h) for h in hx),) if kind == "lstm" \
        else (rnd(hx[0]),), rnd


def _fn(module):
    def f(params, x, *hx):
        y, h = functional_call(module, params, (x, hx[0] if hx else None))
        return (y, *h) if isinstance(h, tuple) else (y, h)
    return f


def _tree(tree, fn):
    return torch.utils._pytree.tree_map(fn, tree)


def _torch_jvp(ref, dtype, x, hx, tx, thx, tp):
    """stock torch on the CPU: (primal outputs, tangents) as float64 numpy, (y, h_n[, c_n])"""
    m = copy.deepcopy(ref).to(dtype)
    p = {n: q.detach() for n, q in m.named_parameters()}
    cast = lambda tree: _tree(tree, lambda t: t.to(dtype))  # noqa: E731
    with torch.backends.mkldnn.flags(enabled=False):
        prim, tan = jvp(_fn(m), (p, x.to(dtype), *cast(hx)), (cast(tp), tx.to(dtype), *cast(thx)))
    return [t.detach().double().numpy() for t in prim], [t.detach().double().numpy() for t in tan]


def _mine(ref):
    import b200rnn

    return b200rnn.from_torch(copy.deepcopy(ref).float()).to(DEV)


def _mine_jvp(mine, x, hx, tx, thx, tp, tf32=False):
    dev = lambda tree: _tree(tree, lambda t: t.float().to(DEV))  # noqa: E731
    p32 = {n: q.detach() for n, q in mine.named_parameters()}
    with _tf32(tf32):
        prim, tan = jvp(_fn(mine), (p32, dev(x), *dev(hx)), (dev(tp), dev(tx), *dev(thx)))
    return [t.detach().cpu().double().numpy() for t in prim], [t.detach().cpu().double().numpy() for t in tan]


def _free_running(ref, x, hx, tx, thx, tp, tf32, kind, relu_check=True):
    """the tangents of stock float64, stock fp32 and the kernels; the calibrated check per tensor"""
    p64, want = _torch_jvp(ref, torch.float64, x, hx, tx, thx, tp)
    p32, t32 = _torch_jvp(ref, torch.float32, x, hx, tx, thx, tp)
    pm, got = _mine_jvp(_mine(ref), x, hx, tx, thx, tp, tf32)
    if kind == "rnn_relu" and relu_check:   # the precondition of the bound: one branch at every element
        for y in (pm[0], p32[0]):
            assert np.array_equal(y > 0, p64[0] > 0), "a relu branch differs from float64"
    scale = 2.0 ** 13 if tf32 else 1.0
    ratios, bad = {}, []
    for k, g, w, t in zip(("y", "h_n", "c_n"), got, want, t32):
        assert g.shape == w.shape, k
        e_k, e_t = _norm_err(g, w), _norm_err(t, w)
        ratios[k] = e_k / max(e_t, 1e-300)
        if not e_k <= 4 * scale * e_t + 1e-6:
            bad.append((k, e_k, e_t))
    return ratios, bad


# ---- batched tangents (M > 1) -----------------------------------------------------------------------------------------

def _batched_case(kind, I, H, L, bi, B, M, group, seed=0):
    """primals, the function of them, and M random tangent directions (a leading [M] on every tangent)"""
    D = 2 if bi else 1
    ref = _stock(kind, I, H, L, bi, "default", seed)
    with torch.no_grad():   # away from default init, as test_gpu_jvp.py
        for p in ref.parameters():
            p.mul_(2.0)
    mine = _mine(ref).eval()
    x, hx, _, _, _ = _inputs(kind, I, H, L, D, B, 12, "default")
    x, hx = x.to(DEV), _tree(hx, lambda t: t.to(DEV))
    p32 = {n: q.detach() for n, q in mine.named_parameters()}
    f = _fn(mine)
    if group == "x":
        prim, fn = (x,), lambda x: f(p32, x, *hx)
    elif group in ("h_0", "c_0"):
        if kind == "lstm":
            h0, c0 = hx[0]
            prim, fn = ((h0,), lambda h: f(p32, x, (h, c0))) if group == "h_0" else ((c0,), lambda c: f(p32, x, (h0, c)))
        else:
            prim, fn = (hx[0],), lambda h: f(p32, x, h)
    elif group == "all":
        prim, fn = (p32, x, *hx), f
    else:
        sub = {n: q for n, q in p32.items() if n.startswith(group)}
        prim, fn = (sub,), lambda s: f({**p32, **s}, x, *hx)
    g = torch.Generator().manual_seed(seed + 9)
    tans = _tree(prim, lambda t: torch.randn((M, *t.shape), generator=g).to(DEV))
    return fn, prim, tans


def _check_batched(fn, prim, tans, M):
    batched = torch.vmap(lambda t: jvp(fn, prim, t)[1])(tans)
    for m in range(M):
        single = jvp(fn, prim, _tree(tans, lambda t: t[m]))[1]
        for b, s in zip(batched, single):
            assert torch.equal(b[m], s), m
    return batched


@pytest.mark.parametrize("group", BATCH_GROUPS)
@pytest.mark.parametrize("name", list(BATCH))
def test_batched_directions_equal_single_directions_bitwise(name, group):
    kind, I, H, L, bi, B, M, _ = BATCH[name]
    if group == "c_0" and kind != "lstm":
        pytest.skip("only the LSTM has a cell state")
    fn, prim, tans = _batched_case(kind, I, H, L, bi, B, M, group)
    batched = _check_batched(fn, prim, tans, M)
    # the directions differ: a direction that read direction 0's tangent would equal it
    assert all(not torch.equal(batched[0][m], batched[0][0]) for m in range(1, M))


def test_batched_directions_beyond_one_wave_bitwise():
    kind, I, H, L, bi, B, M, _ = WAVE
    fn, prim, tans = _batched_case(kind, I, H, L, bi, B, M, "all")
    batched = _check_batched(fn, prim, tans, M)
    assert all(not torch.equal(batched[0][m], batched[0][0]) for m in range(1, M))


@pytest.mark.parametrize("kind", ["gru", "lstm", "rnn_tanh"])
def test_batched_dropout_directions_carry_the_primal_masks(kind):
    """train mode, inter-layer dropout, M = 4 directions of x': each against float64 stock jvp through the layers with
    the Philox masks the primal drew (oracle/philox.py), within 4 x stock fp32's error with the same masks"""
    from oracle import philox
    from test_gpu_jvp import _layer_stack

    L, D, H, T, B, I, p, M = 3, 2, 64, 15, 6, 24, 0.4, 4
    ref = _stock(kind, I, H, L, True, "saturated", dropout=p)
    mine = _mine(ref).train()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(T, B, I, generator=g)
    v = torch.randn(M, T, B, I, generator=g)
    seed, off = (int(t) & (2 ** 64 - 1) for t in mine._rng_state.tolist())
    p32 = {n: q.detach() for n, q in mine.named_parameters()}
    xd = x.to(DEV)
    got = torch.vmap(lambda t: jvp(lambda x: functional_call(mine, p32, (x,))[0], (xd,), (t,))[1])(v.to(DEV))
    got = got.cpu().double().numpy()
    fac = [torch.from_numpy(philox.dropout_factor(seed, off, l, T * B * D * H, p)).double().view(T, B, D * H)
           for l in range(L - 1)]

    def stack(dtype):
        layers = [m.to(dtype) for m in _layer_stack(ref.double(), kind, L, D, I, H)]

        def f(h):
            for l, m in enumerate(layers):
                h = m(h)[0]
                if l < L - 1:
                    h = h * fac[l].to(dtype)
            return h
        return f

    with torch.backends.mkldnn.flags(enabled=False):
        for m in range(M):
            want = jvp(stack(torch.float64), (x.double(),), (v[m].double(),))[1].detach().numpy()
            t32 = jvp(stack(torch.float32), (x,), (v[m],))[1].detach().double().numpy()
            e_k, e_t = _norm_err(got[m], want), _norm_err(t32, want)
            _record_ratio("dropout_err_over_torch32", kind, "saturated", "direction%d" % m, e_k / max(e_t, 1e-300))
            assert e_k <= 4 * e_t + 1e-6, (kind, m, e_k, e_t)


# ---- per-step, teacher forced -----------------------------------------------------------------------------------------

def _w64(ref, d, tp):
    sfx = "_l0" + ("_reverse" if d else "")
    names = [n + sfx for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    return ([getattr(ref, n).detach().double().numpy() for n in names], [tp[n].double().numpy() for n in names])


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("name", list(STEP))
def test_per_step_tangent_within_rounding_bound(name, regime):
    from oracle.rnn_numpy import elman_step_jvp, gru_step_jvp, lstm_step_jvp

    kind, I, H, B, bi, _ = STEP[name]
    regime = _regime(kind, regime)
    I = 1024 if regime == "large_input" else I
    T, D = (120 if regime in ("saturated", "radius") else 40), (2 if bi else 1)
    ref = _stock(kind, I, H, 1, bi, regime)
    x, hx, tx, thx, rnd = _inputs(kind, I, H, 1, D, B, T, regime)
    tp = {n: rnd(p) for n, p in ref.named_parameters()}
    mine = _mine(ref)
    x64, xd64 = x.double().numpy(), tx.double().numpy()
    ws = [_w64(ref, d, tp) for d in range(D)]
    worst = 0.0
    if kind != "lstm":   # one call: the trajectories are y and y'
        (y, _), (yd, _) = _mine_jvp(mine, x, hx, tx, thx, tp)
        h0, h0d = hx[0].double().numpy(), thx[0].double().numpy()
        for d in range(D):
            w, wd = ws[d]
            ys, yds = y[:, :, d * H:(d + 1) * H], yd[:, :, d * H:(d + 1) * H]
            for t in range(T):
                tp_ = t + 1 if d else t - 1
                first = not 0 <= tp_ < T
                hp, hdp = (h0[d], h0d[d]) if first else (ys[tp_], yds[tp_])
                if kind == "gru":
                    want, S = gru_step_jvp(x64[t], hp, *w, xd64[t], hdp, *wd)
                else:
                    want, S = elman_step_jvp(x64[t], hp, *w, xd64[t], hdp, *wd, nonlinearity=kind[4:])
                    if kind == "rnn_relu":
                        a = x64[t] @ w[0].T + w[2] + hp @ w[1].T + w[3]
                        assert np.array_equal(ys[t] > 0, a > 0), (name, regime, d, t, "a relu branch differs")
                worst = max(worst, (np.abs(yds[t] - want) / (KAPPA_T * U32 * S)).max())
    else:   # chained one-step calls through (h, c) and (h', c')
        (h, c), (hd, cd) = hx[0], thx[0]
        for t in range(T):
            (_, h1, c1), (_, h1d, c1d) = _mine_jvp(mine, x[t:t + 1], ((h, c),), tx[t:t + 1], ((hd, cd),), tp)
            hp, cp, hdp, cdp = (a.double().numpy() for a in (h, c, hd, cd))
            for d in range(D):
                w, wd = ws[d]
                want_h, want_c, S_h, S_c = lstm_step_jvp(x64[t], hp[d], cp[d], *w, xd64[t], hdp[d], cdp[d], *wd)
                for got, want, S in ((h1d[d], want_h, S_h), (c1d[d], want_c, S_c)):
                    worst = max(worst, (np.abs(got - want) / (KAPPA_T * U32 * S)).max())
            h, c, hd, cd = (torch.from_numpy(a).float() for a in (h1, c1, h1d, c1d))
    _record_ratio("per_step_max_err_over_bound", name, regime, "T%d" % T, worst)
    if regime != "small_signal":
        assert worst <= 1.0, (name, regime, worst)


# ---- free running, calibrated against torch fp32 ----------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["fp32", "tf32"])
@pytest.mark.parametrize("name", list(FREE))
def test_free_running_tangent_vs_f64(name, mode):
    kind, I, H, L, bi, B, T, regime = FREE[name]
    D = 2 if bi else 1
    ref = _stock(kind, I, H, L, bi, regime)
    x, hx, tx, thx, rnd = _inputs(kind, I, H, L, D, B, T, regime)
    tp = {n: rnd(p) for n, p in ref.named_parameters()}
    ratios, bad = _free_running(ref, x, hx, tx, thx, tp, mode == "tf32", kind)
    for k, v in ratios.items():
        _record_ratio("free_running_err_over_torch32", name, regime + "_" + mode, k, v)
    assert not bad, (name, mode, bad)


@pytest.mark.parametrize("name", PRIMAL)
def test_tangent_of_every_saving_primal_config_vs_f64(name):
    """the tangent kernel on the reserve each fixed forward config writes (the configs: see the child-process test)"""
    kind, I, H, B, bi, _, mode = FIXED_CONFIGS[name]
    D, T = (2 if bi else 1), 24
    ref = _stock(kind, I, H, 1, bi, "saturated")
    x, hx, tx, thx, rnd = _inputs(kind, I, H, 1, D, B, T, "saturated")
    tp = {n: rnd(p) for n, p in ref.named_parameters()}
    ratios, bad = _free_running(ref, x, hx, tx, thx, tp, mode == "tf32", kind)
    for k, v in ratios.items():
        _record_ratio("primal_config_err_over_torch32", name, "saturated_" + mode, k, v)
    assert not bad, (name, bad)


EDGES = {"T1": dict(T=1, B=5), "B1": dict(T=20, B=1), "unbatched": dict(T=20, B=1, unbatched=True)}


@pytest.mark.parametrize("edge", list(EDGES))
@pytest.mark.parametrize("kind", ["gru", "lstm", "rnn_tanh"])
def test_edge_shapes_vs_f64(kind, edge):
    """T = 1: the first step's W_hh' h_0 GEMM alone; B = 1; unbatched x and hx"""
    e = EDGES[edge]
    I, H, L, D = 40, 96, 2, 2
    ref = _stock(kind, I, H, L, True, "saturated")
    x, hx, tx, thx, rnd = _inputs(kind, I, H, L, D, e["B"], e["T"], "saturated", e.get("unbatched", False))
    tp = {n: rnd(p) for n, p in ref.named_parameters()}
    ratios, bad = _free_running(ref, x, hx, tx, thx, tp, False, kind)
    for k, v in ratios.items():
        _record_ratio("edge_err_over_torch32", kind, edge, k, v)
    assert not bad, (kind, edge, bad)


@pytest.mark.parametrize("with_state_dots", [True, False], ids=["dots", "no_dots"])
@pytest.mark.parametrize("BT", [(0, 6), (4, 0)], ids=["B0", "T0"])
@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_empty_call_passes_the_initial_tangents_through(kind, BT, with_state_dots):
    """b200rnn_forward_tangent with B == 0 or T == 0 and M = 3 directions: h_n' (c_n') is h_0' (c_0') of each direction,
    or 0 when it is NULL"""
    from b200rnn.functional import _rnn_tangent_impl

    B, T = BT
    M, I, H, L, D = 3, 24, 48, 2, 2
    mine = _mine(_stock(kind, I, H, L, True, "default"))
    cfg = mine._config()
    g = torch.Generator().manual_seed(11)
    rnd = lambda *s: torch.randn(*s, generator=g).to(DEV)  # noqa: E731
    x_tm, y = rnd(T, B, I), rnd(T, B, D * H)
    reserve = torch.zeros(256, dtype=torch.uint8, device=DEV)
    h_0, c_0 = rnd(L * D, B, H), (rnd(L * D, B, H) if kind == "lstm" else None)
    h0d = rnd(M, L * D, B, H) if with_state_dots else None
    c0d = rnd(M, L * D, B, H) if with_state_dots and kind == "lstm" else None
    # NaN in the memory the allocator hands out next: the call must write every element of h_n' / c_n'
    junk = [torch.full((M * L * D * B * H,), float("nan"), device=DEV) for _ in range(2)]
    del junk
    y_dot, hnd, cnd = _rnn_tangent_impl(cfg, x_tm, y, reserve, h_0, c_0, mine._flat_weights, rnd(M, T, B, I), h0d, c0d,
                                        [None] * len(mine._flat_weights), directions=M)
    torch.cuda.synchronize()
    assert y_dot.shape == (M, T, B, D * H) and hnd.shape == (M, L * D, B, H)
    assert torch.equal(hnd, h0d if with_state_dots else torch.zeros_like(hnd))
    if kind == "lstm":
        assert torch.equal(cnd, c0d if with_state_dots else torch.zeros_like(cnd))
    else:
        assert cnd is None


# ---- configs and tiers reached (B200RNN_DEBUG is read once per process) -------------------------------------------------

_CHILD = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}, {tests!r}]
import torch
import test_gpu_jvp_numerics_f64 as J
from test_gpu_anyh_numerics_f64 import _tf32
from torch.func import jvp
for name in J.PRIMAL:
    kind, I, H, B, bi, _, mode = J.FIXED_CONFIGS[name]
    ref = J._stock(kind, I, H, 1, bi, "saturated")
    x, hx, tx, thx, rnd = J._inputs(kind, I, H, 1, 2 if bi else 1, B, 3, "saturated")
    J._mine_jvp(J._mine(ref), x, hx, tx, thx, {{n: rnd(p) for n, p in ref.named_parameters()}}, mode == "tf32")
    torch.cuda.synchronize()
    print("[b200rnn] ran primal", name, file=sys.stderr, flush=True)
for name, (kind, I, H, B, bi, tier) in J.STEP.items():
    ref = J._stock(kind, I, H, 1, bi, "default")
    x, hx, tx, thx, rnd = J._inputs(kind, I, H, 1, 2 if bi else 1, B, 3, "default")
    J._mine_jvp(J._mine(ref), x, hx, tx, thx, {{n: rnd(p) for n, p in ref.named_parameters()}})
    torch.cuda.synchronize()
    print("[b200rnn] ran step", name, file=sys.stderr, flush=True)
for name, (kind, I, H, L, bi, B, M, tier) in list(J.BATCH.items()) + [("wave", J.WAVE)]:
    for m in (1, M):
        fn, prim, tans = J._batched_case(kind, I, H, L, bi, B, m, "all")
        torch.vmap(lambda t: jvp(fn, prim, t)[1])(tans)
        torch.cuda.synchronize()
        print("[b200rnn] ran batch", name, m, file=sys.stderr, flush=True)
"""


@pytest.fixture(scope="module")
def debug_lines():
    env = dict(os.environ, B200RNN_DEBUG="1")
    code = _CHILD.format(root=ROOT, pkg=PKG, tests=os.path.join(ROOT, "tests"))
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout + proc.stderr[-4000:]
    runs, pending = {}, []
    for ln in proc.stderr.splitlines():
        if not ln.startswith("[b200rnn] "):
            continue
        body = ln[len("[b200rnn] "):]
        if body.startswith("ran "):
            runs[tuple(body.split()[1:])] = pending
            pending = []
        elif body.startswith(("fwd cfg", "fwd anyh cfg", "fwd elman cfg", "tan ")):
            pending.append(body.split(":")[0])
    return runs


def test_child_reaches_every_primal_config_and_its_tangent_launch(debug_lines):
    for name in PRIMAL:
        kind, I, H, B, bi, _, _ = FIXED_CONFIGS[name]
        lines = debug_lines[("primal", name)]
        assert FWD_LINE[name] in lines, (name, lines)
        tan = [ln for ln in lines if ln.startswith("tan ")]
        assert len(tan) == 1 and f"cfg {MODE_NAME[kind]} VL=0 H={H} " in tan[0], (name, lines)


def test_child_reaches_every_tier_and_the_launch_shape_does_not_depend_on_M(debug_lines):
    seen = set()
    for name, (kind, I, H, B, bi, tier) in STEP.items():
        tan = [ln for ln in debug_lines[("step", name)] if ln.startswith("tan ")]
        assert len(tan) == 1 and f"cfg {MODE_NAME[kind]} VL=0 H={H} " in tan[0] and f"tier={tier}" in tan[0], (name, tan)
        seen.add((kind, tier))
    assert seen == {(k, t) for k in MODE_NAME for t in ("smem", "l2")}, seen
    for name, (kind, I, H, L, bi, B, M, tier) in list(BATCH.items()) + [("wave", WAVE)]:
        one = [ln for ln in debug_lines[("batch", name, "1")] if ln.startswith("tan ")]
        many = [ln for ln in debug_lines[("batch", name, str(M))] if ln.startswith("tan ")]
        assert len(one) == len(many) == L and all(f"tier={tier}" in ln for ln in one), (name, one, many)
        assert one == many, (name, one, many)   # the same cluster shape and tier, whatever M
