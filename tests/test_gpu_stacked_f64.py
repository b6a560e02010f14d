"""Stacked GRU / LSTM / RNN calls: each layer bitwise a one-layer call, and the whole stack against float64 off default init.

The float64 files (test_gpu_numerics_f64.py, test_gpu_anyh_numerics_f64.py, test_gpu_h16_numerics_f64.py) build one-layer
modules. A stacked call runs code no one-layer call reaches (csrc/api.cu): layer l > 0 projects layer l - 1's output from
the reserve (saving) or from the ping-pong scratch (no-grad, L = 3 reuses a buffer), the inter-layer dropout runs in
place when nothing is saved, the backward's dX GEMM of layer l writes the dy of layer l - 1 into scratch (the second
direction accumulating into it) and the dropout backward runs in place on it, dW_ih of layer l reads the dropped output,
and the states are per-layer slices. Layer l > 0 projects with K = D * HO: 2048 for a bidirectional H = 1024 stack.

1. Chain identity (bitwise). In api.cu each layer of a stacked call uses the plan, GEMM and recurrence a one-layer call
   uses on the same values: the fp32-A projection route is bitwise the presplit route (test_gpu_gemm_f32a.py) and the
   inner padding rows are +0 in both. So an L-layer call must equal a chain of L one-layer calls on the same weights,
   bit for bit, where layer l of the chain takes the library's own output of layer l - 1 dropped exactly as
   dropout_kernel drops it: torch.where(keep, y * scale, 0), keep and scale from oracle.philox keyed by the stacked
   call's rng_state with stream = l. The chain's backward is autograd of that expression. Checked: y, every h_n / c_n
   slice, dx, every layer's dW_ih / dW_hh / db_ih / db_hh / dW_hr, every dh_0 / dc_0 slice, with random loss weights on y
   and on each state slice. Cases: every fixed plan-table family, the runtime-sized GRU / LSTM / RNN in both weight
   tiers (with bidirectional H = 1008 / 1024 stacks, inner K = 2016 / 2048), L = 3 ragged with hx and dropout,
   batch_first, more batch rows than one wave of clusters, T = 1, a loss on an inner layer's state only; saving
   forward + backward, the no-grad train-mode forward at L = 3, TF32 mode, the 16-bit forward (round -> dropout ->
   round between layers; its backward keeps the inner dy in fp32 by design and stays with test_gpu_h16_modules.py),
   and the no-grad fused entry on the benchmark's encoders (audio GRU-256 x 2 with LayerNorm and the weight cache, text
   BiLSTM-128 x 2 at I = 1024). A subset runs on the NaN-filled allocator of test_gpu_poisoned_buffers.py. A
   B200RNN_DEBUG child process checks that each layer's x-projection and recurrence config lines are those of its
   chain, that an inner layer reaches every fixed plan entry, and that a tensor-core x-projection with K = 2048 runs.

2. Against float64. Free running: y, the states and every gradient of every layer, normwise, within
   4 * err_torch32 + 1e-6 (TF32 mode: err_torch32 x 2^13) as in test_gpu_numerics_f64.py, where the float64 and the
   stock fp32 references are chains of stock one-layer modules with the same dropout masks (oracle/stacked.py), at
   L = 2 and 3, ragged, with hx and dropout, in the default, saturated (relu: radius) and large_input regimes; the
   fused no-grad y_pool of the benchmark encoders in the saturated regime. Per step: given part 1, the teacher-forced
   check of test_gpu_numerics_f64.py applies to each layer of the chain with the kernel's own dropped output of the
   layer below as x; it runs on the inner layer of bidirectional GRU-1024 / LSTM-1008 stacks and of one fixed config
   per family, with the bound KAPPA(K) u S below.

KAPPA(K), counted as in test_gpu_numerics_f64.py: 4 roundings at the pre-activation's magnitude (the input-projection
accumulator, its bias, the recurrent accumulator, the combine), plus the accumulation chain of the input-projection
GEMM with k-blocks of 8, depth K / 8, which errs by sqrt(K / 8) u |terms| with high probability (Higham & Mary, SIAM J.
Sci. Comput. 41(5), 2019), plus 8 for the activations and the cell update:

    KAPPA(K) = 4 + ceil(sqrt(K / 8)) + 8        24 at K <= 1024 (the one-layer files' KAPPA), 26 at 2016, 28 at 2048

The constant is derived, not fitted. B200RNN_NUMERICS_RECORD=<path> writes the ratios to stacked_f64_results.json beside
<path>."""
import contextlib
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import philox
from oracle.stacked import chained, split_layers
from test_gpu_numerics_f64 import CONFIGS as FIXED
from test_gpu_numerics_f64 import BWD_LINE, FWD_LINE, U32, _input, _norm_err, _ragged_lengths
from test_gpu_numerics_f64 import KAPPA as KAPPA_1024
from test_gpu_poisoned_buffers import POISON, _FilledTorch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
RECORDS = {}
SEED, OFFSET = 0x5EED5, 777


def kappa(K):
    return 4 + math.ceil(math.sqrt(K / 8)) + 8


assert kappa(1024) == KAPPA_1024 and kappa(2048) == 28

# name -> kind, I, H, B, bidirectional, proj_size, mode ("fp32" or "tf32"): the fixed plan-table families at the batch
# sizes of test_gpu_numerics_f64.CONFIGS, then the runtime-sized kernels in both weight tiers
CONFIGS = {n: c for n, c in FIXED.items() if c[6] != "f16"}
CONFIGS.update({
    "gru_h272_bi": ("gru", 64, 272, 24, True, 0, "fp32"),
    "gru_h1024_bi": ("gru", 64, 1024, 6, True, 0, "fp32"),        # inner K = 2048 on the tensor cores
    "lstm_h96_bi": ("lstm", 40, 96, 40, True, 0, "fp32"),
    "lstm_h1008_bi": ("lstm", 48, 1008, 4, True, 0, "fp32"),      # inner K = 2016 on the FFMA GEMM
    "tanh_h272": ("rnn_tanh", 40, 272, 16, False, 0, "fp32"),
    "tanh_h1008_bi": ("rnn_tanh", 64, 1008, 8, True, 0, "fp32"),
    "relu_h464_bi": ("rnn_relu", 64, 464, 16, True, 0, "fp32"),
    "relu_h1024": ("rnn_relu", 48, 1024, 6, False, 0, "fp32"),
})
STATES = {"gru": ("h_n",), "lstm": ("h_n", "c_n"), "rnn_tanh": ("h_n",), "rnn_relu": ("h_n",)}


@pytest.fixture(scope="module", autouse=True)
def _record():
    yield
    path = os.environ.get("B200RNN_NUMERICS_RECORD")
    if path and RECORDS:
        with open(os.path.join(os.path.dirname(os.path.abspath(path)), "stacked_f64_results.json"), "w") as f:
            json.dump(RECORDS, f, indent=1, sort_keys=True)
            f.write("\n")


def _record_ratio(kind, name, regime, key, value):
    RECORDS.setdefault(kind, {}).setdefault(name, {}).setdefault(regime, {})[key] = float(value)


# ---- models ---------------------------------------------------------------------------------------------------------

def _stock(kind, I, H, L, bi, P=0, dropout=0.0):
    if kind in ("gru", "lstm"):
        cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
        return cls(I, H, num_layers=L, bidirectional=bi, dropout=dropout, **({"proj_size": P} if P else {}))
    return torch.nn.RNN(I, H, num_layers=L, nonlinearity=kind[4:], bidirectional=bi, dropout=dropout)


def _stack_model(kind, I, H, L, bi, P, regime, dropout=0.0, seed=0):
    """stock L-layer module (fp32, CPU) with the regime's weights in every layer (test_gpu_numerics_f64._torch_model;
    radius: each W_hh at spectral radius 0.95, test_gpu_anyh_numerics_f64._torch_model)"""
    torch.manual_seed(seed)
    ref = _stock(kind, I, H, L, bi, P, dropout)
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
            elif regime == "radius" and n.startswith("weight_hh"):
                p.mul_(0.95 / max(abs(np.linalg.eigvals(p.double().numpy()))))
    return ref


def _cfg(mod, tf32, training=None, dropout=None):
    cfg = mod._config()
    cfg.tf32 = tf32
    if training is not None:
        cfg.training = training
    if dropout is not None:
        cfg.dropout = dropout
    return cfg


def _drop_args(T, B, W, p, layer, rng0, batch_first=False):
    """(keep, scale) of dropout_kernel's mask of `layer` for a call that started from rng_state rng0, laid out [T,B,W]
    (or [B,T,W])"""
    keep = philox.keep_mask(int(rng0[0]), int(rng0[1]), layer, T * B * W, p).reshape(T, B, W)
    keep = torch.from_numpy(keep).to(DEV)
    if batch_first:
        keep = keep.transpose(0, 1)
    return keep, torch.tensor(philox.scale(p), dtype=torch.float32, device=DEV)


def _dropped(y, keep, scale):
    """dropout_kernel's expression, in y's dtype (16-bit: widened, scaled in fp32 and rounded again)"""
    return torch.where(keep, y.float() * scale, torch.zeros((), device=y.device)).to(y.dtype)


# ---- one case: the stacked call and its chain -------------------------------------------------------------------------

@contextlib.contextmanager
def _allocator(word):
    """functional.py's torch.empty / empty_like filled with `word` (None: torch's own)"""
    from b200rnn import functional

    if word is None:
        yield
        return
    saved = functional.torch
    functional.torch = _FilledTorch(word)
    try:
        yield
    finally:
        functional.torch = saved


def _call(mod, cfg, x, rng, lens, hx):
    from b200rnn.functional import rnn_forward

    out = rnn_forward(x, mod._flat_weights, cfg, rng, lengths=lens, hx=hx)
    return out[0], list(out[1:])


def _mark(on, side):
    """B200RNN_DEBUG child: the route lines that follow belong to `side`"""
    if on:
        print("[b200rnn] side", side, file=sys.stderr, flush=True)


def _run_case(kind, I, H, B, bi, P=0, *, L=2, T=10, mode="fp32", dtype=torch.float32, ragged=False, hx=True, p=0.0,
              grad=True, save=False, batch_first=False, inner_loss=False, fill=None, seed=0, route_marks=False):
    """the stacked call and its chain on the same inputs: {"stack": {name: tensor}, "chain": {...}}. `grad`: forward
    and backward; `save`: the saving forward alone (x requires grad, no backward)"""
    import b200rnn

    tf32 = mode == "tf32"
    ref = _stack_model(kind, I, H, L, bi, P, "default", dropout=p, seed=seed)
    D, HO = (2 if bi else 1), (P or H)
    W = D * HO
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(T, B, I, generator=g)
    lens = None
    if ragged:
        lens = _ragged_lengths(B, T)
        lens[1 % B] = 1   # lengths 1 and T present
    st0 = [0.5 * torch.randn(L * D, B, HO, generator=g)] + (
        [0.5 * torch.randn(L * D, B, H, generator=g)] if kind == "lstm" else [])
    wy = torch.randn(T, B, W, generator=g)
    ws = [torch.randn(s.shape, generator=g) for s in st0]
    if inner_loss:   # only the states of layer 0 reach the loss
        wy = torch.zeros_like(wy)
        ws = [torch.cat([w[:D], torch.zeros_like(w[D:])]) for w in ws]
    if batch_first:
        x, wy = x.transpose(0, 1).contiguous(), wy.transpose(0, 1).contiguous()
    stack = b200rnn.from_torch(ref).to(DEV, dtype).train(p > 0)
    if batch_first:
        stack.batch_first = True
    layers = [b200rnn.from_torch(m).to(DEV, dtype).train(p > 0) for m in split_layers(ref)]
    rng0 = (SEED + seed, OFFSET)
    res = {}
    track = grad or save
    with _allocator(fill), torch.set_grad_enabled(track):
        # the stacked call
        _mark(route_marks, "stack")
        xs = x.to(DEV, dtype).requires_grad_(track)
        hs = [s.to(DEV, dtype).requires_grad_(track) for s in st0] if hx else []
        h_in = None if not hx else (tuple(hs) if kind == "lstm" else hs[0])
        rng = torch.tensor(rng0, dtype=torch.int64, device=DEV)
        y, sts = _call(stack, _cfg(stack, tf32), xs, rng, lens, h_in)
        out = {"y": y, **dict(zip(STATES[kind], sts))}
        if grad:
            (sum((v.float() * w.to(DEV)).sum() for v, w in zip((y, *sts), (wy, *ws)))).backward()
            out["dx"] = xs.grad
            out.update({"d" + n: q.grad for n, q in stack.named_parameters()})
            out.update(dict(zip(("dh_0", "dc_0"), (s.grad for s in hs))))
        res["stack"] = out
        # the chain
        _mark(route_marks, "chain")
        xc = x.to(DEV, dtype).requires_grad_(track)
        hc = [s.to(DEV, dtype).requires_grad_(track) for s in st0] if hx else []
        h = xc
        finals = []
        for l, m in enumerate(layers):
            first, last = l == 0, l == L - 1
            if batch_first and l == 1:   # the stack's inner layers are time-major, as api.cu keeps them
                h = h.transpose(0, 1).contiguous()
            m.batch_first = batch_first and first
            h_l = None if not hx else tuple(s[l * D:(l + 1) * D] for s in hc)
            h_l = None if h_l is None else (h_l if kind == "lstm" else h_l[0])
            h, s_l = _call(m, _cfg(m, tf32), h, None, lens, h_l)
            finals.append(s_l)
            if not last and p > 0:
                Tl, Bl = (h.shape[1], h.shape[0]) if (batch_first and first) else h.shape[:2]
                keep, scale = _drop_args(Tl, Bl, W, p, l, rng0, batch_first and first)
                h = _dropped(h, keep, scale)
        if batch_first and L > 1:
            h = h.transpose(0, 1)
        sts_c = [torch.cat([f[i] for f in finals]) for i in range(len(finals[0]))]
        outc = {"y": h, **dict(zip(STATES[kind], sts_c))}
        if grad:
            (sum((v.float() * w.to(DEV)).sum() for v, w in zip((h, *sts_c), (wy, *ws)))).backward()
            outc["dx"] = xc.grad
            for l, m in enumerate(layers):
                outc.update({"d" + n.replace("_l0", f"_l{l}"): q.grad for n, q in m.named_parameters()})
            outc.update(dict(zip(("dh_0", "dc_0"), (s.grad for s in hc))))
        res["chain"] = outc
        torch.cuda.synchronize()
    assert int(rng[1]) == OFFSET + ((T * B * W + 3) // 4 if p > 0 and stack.training else 0)
    return {k: {n: t.detach().clone() for n, t in v.items()} for k, v in res.items()}


def _assert_bitwise(res, what):
    a, b = res["stack"], res["chain"]
    assert sorted(a) == sorted(b), (what, sorted(a), sorted(b))
    bad = [k for k in a if not torch.equal(a[k], b[k])]
    assert not bad, (what, [(k, (a[k].double() - b[k].double()).abs().max().item()) for k in bad])


# ---- 1. chain identity ------------------------------------------------------------------------------------------------

def _chain_cases():
    cases = {}
    for name, (kind, I, H, B, bi, P, mode) in CONFIGS.items():
        cases[f"{name}-L2"] = dict(kind=kind, I=I, H=H, B=B, bi=bi, P=P, mode=mode)
    for name in ("gru256_bs4", "gru256_tc8_3xtf32", "bilstm128", "bilstmp_h256_p64", "gru_h272_bi", "lstm_h96_bi",
                 "tanh_h1008_bi", "relu_h464_bi", "gru_h1024_bi"):
        kind, I, H, B, bi, P, mode = CONFIGS[name]
        cases[f"{name}-L3-ragged-hx-drop"] = dict(kind=kind, I=I, H=H, B=B, bi=bi, P=P, mode=mode, L=3, ragged=True,
                                                  p=0.3)
    cases["bilstm256-L2-batch_first-drop"] = dict(kind="lstm", I=256, H=256, B=32, bi=True, batch_first=True, p=0.3)
    cases["lstm_h96_bi-L2-batch_first-ragged"] = dict(kind="lstm", I=40, H=96, B=40, bi=True, batch_first=True,
                                                      ragged=True)
    # more batch rows than one wave of co-resident clusters
    cases["gru256-L2-B512"] = dict(kind="gru", I=256, H=256, B=512, bi=False, T=6)
    cases["gru_h272_bi-L2-B600-drop"] = dict(kind="gru", I=64, H=272, B=600, bi=True, T=6, p=0.3)
    cases["gru256_bs4-L2-T1"] = dict(kind="gru", I=256, H=256, B=64, bi=False, T=1, p=0.3)
    cases["lstm_h464_bi-L2-T1"] = dict(kind="lstm", I=64, H=464, B=12, bi=True, T=1)
    cases["bilstm128-L3-inner_loss"] = dict(kind="lstm", I=256, H=128, B=16, bi=True, L=3, inner_loss=True)
    cases["gru_h272_bi-L2-inner_loss"] = dict(kind="gru", I=64, H=272, B=24, bi=True, inner_loss=True)
    cases["bilstm128-L3-tf32-drop"] = dict(kind="lstm", I=256, H=128, B=16, bi=True, L=3, mode="tf32", p=0.3,
                                           ragged=True)
    cases["gru_h1024_bi-L2-tf32"] = dict(kind="gru", I=64, H=1024, B=6, bi=True, mode="tf32")
    return cases


CHAIN = _chain_cases()


@pytest.mark.parametrize("case", list(CHAIN))
def test_stacked_call_is_a_chain_of_one_layer_calls(case):
    _assert_bitwise(_run_case(**CHAIN[case]), case)


NOGRAD = {
    "gru256_bs4": ("gru", 256, 256, 64, False, 0),
    "gru256_tc8": ("gru", 256, 256, 128, False, 0),
    "bilstm128_wide": ("lstm", 256, 128, 136, True, 0),
    "bilstmp_h128_p32": ("lstm", 256, 128, 16, True, 32),
    "lstm_h464_bi": ("lstm", 64, 464, 12, True, 0),
    "tanh_h272": ("rnn_tanh", 40, 272, 16, False, 0),
    "gru_h1024_bi": ("gru", 64, 1024, 6, True, 0),
}


@pytest.mark.parametrize("ragged", [False, True], ids=["fixed", "ragged"])
@pytest.mark.parametrize("name", list(NOGRAD))
def test_nograd_three_layers_with_dropout_is_a_chain(name, ragged):
    """no-grad train-mode forward at L = 3: inner outputs in the ping-pong scratch, the dropout in place"""
    kind, I, H, B, bi, P = NOGRAD[name]
    _assert_bitwise(_run_case(kind, I, H, B, bi, P, L=3, ragged=ragged, p=0.3, grad=False), (name, ragged))


H16 = {
    "gru256": ("gru", 256, 256, 64, False),
    "bilstm128": ("lstm", 256, 128, 16, True),
    "lstm_h464_bi": ("lstm", 64, 464, 12, True),
    "tanh_h272_bi": ("rnn_tanh", 40, 272, 16, True),
    "relu_h1024": ("rnn_relu", 48, 1024, 6, False),
}


@pytest.mark.parametrize("saving", [False, True], ids=["nograd", "saving"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", list(H16))
def test_16bit_forward_is_a_chain(name, dtype, saving):
    """the 16-bit forward: an inner output is rounded, dropped in fp32 and rounded again (the saving forward keeps the
    fp32 widening for the backward, which is not compared here)"""
    kind, I, H, B, bi = H16[name]
    res = _run_case(kind, I, H, B, bi, L=3, dtype=dtype, ragged=True, p=0.3, grad=False)
    _assert_bitwise(res, (name, dtype))
    if saving:   # x requires grad: the saving forward, forward only
        res = _run_case(kind, I, H, B, bi, L=2, dtype=dtype, p=0.3, grad=False, save=True)
        _assert_bitwise(res, (name, dtype, "saving"))


POISONED = ["gru256_tc8_3xtf32-L2", "bilstmp_h128_p32-L2", "bilstm128-L3-ragged-hx-drop", "gru_h1024_bi-L3-ragged-hx-drop",
            "relu_h464_bi-L3-ragged-hx-drop", "gru256_bs4-L2-T1"]


@pytest.mark.parametrize("case", POISONED)
def test_chain_on_poisoned_buffers(case):
    """every buffer functional.py allocates filled with a NaN word, then with 0: finite, bitwise equal, and the stack
    still the chain"""
    dirty = _run_case(**CHAIN[case], fill=POISON)
    clean = _run_case(**CHAIN[case], fill=0)
    for side in ("stack", "chain"):
        for k, v in clean[side].items():
            assert torch.isfinite(dirty[side][k]).all(), (case, side, k)
            assert torch.equal(dirty[side][k], v), (case, side, k)
    _assert_bitwise(dirty, case)


# ---- the fused no-grad entry on the benchmark's encoders ------------------------------------------------------------

# name -> kind, I, H, B, T, bidirectional, LayerNorm
ENCODERS = {"audio_gru256": ("gru", 256, 256, 128, 120, False, True),
            "text_bilstm128": ("lstm", 1024, 128, 128, 30, True, False)}


def _fused_case(name, regime="default", p=0.3, route_marks=False):
    """the stacked fused call (y_pool, y, h_n [, c_n]) and a chain of one-layer fused calls, layer 0 with the LayerNorm
    prologue, every call with its weight cache"""
    import b200rnn
    from b200rnn.functional import prepare_weights, rnn_forward_fused

    kind, I, H, B, T, bi, ln = ENCODERS[name]
    D = 2 if bi else 1
    ref = _stack_model(kind, I, H, 2, bi, 0, regime, dropout=p)
    x = _input("saturated" if regime == "saturated" else "default", T, B, I, seed=11)
    g = torch.Generator().manual_seed(12)
    ln_w = (1 + 0.1 * torch.randn(I, generator=g)).to(DEV) if ln else None
    ln_b = (0.1 * torch.randn(I, generator=g)).to(DEV) if ln else None
    stack = b200rnn.from_torch(ref).to(DEV).train()
    layers = [b200rnn.from_torch(m).to(DEV).train() for m in split_layers(ref)]
    rng0 = (SEED, OFFSET)
    xd = x.to(DEV)
    out = {}
    cfg = _cfg(stack, False)
    wc = prepare_weights(stack._flat_weights, cfg)
    for pool in (True, False):
        _mark(route_marks, "stack" if pool else "other")
        rng = torch.tensor(rng0, dtype=torch.int64, device=DEV)
        r = rnn_forward_fused(xd, stack._flat_weights, cfg, rng, ln_w, ln_b, pool_sum=pool, wcache=wc)
        out["stack_pool" if pool else "stack_y"] = r[0]
        out["stack_states"] = list(r[1:])
    _mark(route_marks, "chain")
    c0, c1 = (_cfg(m, False) for m in layers)
    r0 = rnn_forward_fused(xd, layers[0]._flat_weights, c0, None, ln_w, ln_b,
                           wcache=prepare_weights(layers[0]._flat_weights, c0))
    keep, scale = _drop_args(T, B, D * H, p, 0, rng0)
    x1 = _dropped(r0[0], keep, scale)
    wc1 = prepare_weights(layers[1]._flat_weights, c1)
    r1 = rnn_forward_fused(x1, layers[1]._flat_weights, c1, None, pool_sum=True, wcache=wc1)
    _mark(route_marks, "other")
    out["chain_pool"] = r1[0]
    out["chain_y"] = rnn_forward_fused(x1, layers[1]._flat_weights, c1, None, wcache=wc1)[0]
    out["chain_states"] = [torch.cat([a, b]) for a, b in zip(r0[1:], r1[1:])]
    torch.cuda.synchronize()
    return ref, x, ln_w, ln_b, out


@pytest.mark.parametrize("name", list(ENCODERS))
def test_fused_encoder_stack_is_a_chain_of_fused_calls(name):
    _, _, _, _, out = _fused_case(name)
    assert torch.equal(out["stack_pool"], out["chain_pool"]), name
    assert torch.equal(out["stack_y"], out["chain_y"]), name
    for a, b in zip(out["stack_states"], out["chain_states"]):
        assert torch.equal(a, b), name


@pytest.mark.parametrize("name", list(ENCODERS))
def test_fused_encoder_pool_saturated_vs_f64(name):
    """y_pool and the states of the fused no-grad stack (dropout 0.3) against the float64 chain with the same masks,
    within 4 x stock fp32's error"""
    kind, I, H, B, T, bi, ln = ENCODERS[name]
    D, p = (2 if bi else 1), 0.3
    ref, x, ln_w, ln_b, out = _fused_case(name, "saturated", p)
    mask = torch.from_numpy(philox.dropout_factor(SEED, OFFSET, 0, T * B * D * H, p).reshape(T, B, D * H))
    got = {"y_pool": out["stack_pool"], **dict(zip(STATES[kind], out["stack_states"]))}
    refs = {}
    for dt in (torch.float64, torch.float32):
        xx = x.to(dt)
        if ln:
            xx = torch.nn.functional.layer_norm(xx, (I,), ln_w.cpu().to(dt), ln_b.cpu().to(dt), 1e-5)
        with torch.no_grad():
            y, sts = chained(split_layers(_copy(ref).to(dt)), xx, masks=[mask.to(dt)])
        refs[dt] = {"y_pool": y.sum(0), **dict(zip(STATES[kind], sts))}
    bad = []
    for k, want in refs[torch.float64].items():
        e_k, e_t = _norm_err(got[k].cpu(), want), _norm_err(refs[torch.float32][k], want)
        _record_ratio("fused_err_over_torch32", name, "saturated", k, e_k / max(e_t, 1e-300))
        if not e_k <= 4 * e_t + 1e-6:
            bad.append((k, e_k, e_t))
    assert not bad, (name, bad)


def _copy(ref):
    import copy
    return copy.deepcopy(ref)


# ---- routes -----------------------------------------------------------------------------------------------------------

ROUTE_CASES = {k: CHAIN[k] for k in CHAIN if k.endswith("-L2") or k.endswith("-L3-ragged-hx-drop")}

_CHILD = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}, {tests!r}]
import torch
torch.backends.cuda.matmul.fp32_precision = "ieee"
import test_gpu_stacked_f64 as t
for name, case in {cases!r}.items():
    print("[b200rnn] case", name, file=sys.stderr, flush=True)
    t._run_case(**dict(case, T=4), route_marks=True)
for name in t.ENCODERS:
    print("[b200rnn] fused", name, file=sys.stderr, flush=True)
    t._fused_case(name, route_marks=True)
"""
_A_ROUTE = re.compile(r" a=\w+$")
_ROUTE = re.compile(r"^\[b200rnn\] ((forward|ffma) x-projection: .*|(fwd|bwd) .*cfg [^:]*)")


def _parse_routes(stderr):
    """{(case, side): [route lines in order]}, side = stack / chain (marked by the child)"""
    routes, key = {}, None
    for ln in stderr.splitlines():
        if ln.startswith("[b200rnn] case ") or ln.startswith("[b200rnn] fused "):
            case = ln.split()[2]
            continue
        if ln.startswith("[b200rnn] side "):
            key = (case, ln.split()[2])
            routes[key] = []
            continue
        mt = _ROUTE.match(ln)
        if mt and key is not None:
            routes[key].append(mt.group(1).split(": need")[0])
    return routes


def test_routes_each_layer_as_its_chain_and_every_fixed_entry_inner():
    env = dict(os.environ, B200RNN_DEBUG="1")
    code = _CHILD.format(root=ROOT, pkg=PKG, tests=os.path.join(ROOT, "tests"), cases=ROUTE_CASES)
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout + proc.stderr[-4000:]
    routes = _parse_routes(proc.stderr)
    cases = list(ROUTE_CASES) + list(ENCODERS)
    inner_fwd, inner_bwd, k2048 = set(), set(), False
    for case in cases:
        stack, chain = routes[(case, "stack")], routes[(case, "chain")]
        # One deliberate difference, in where the x-projection's A operand comes from, not in what the GEMM computes
        # (the case above is bitwise): the stack's inner layer hands the GEMM its dense [T*B, K] output, which one 2-D
        # map reads in place, while a one-layer call describes its caller's x as T steps of B rows, a 3-D map that
        # make_a_f32_map refuses when B neither divides nor is a multiple of the tile's rows (B = 272): the chain
        # gathers a dense copy first.
        assert stack and [_A_ROUTE.sub("", r) for r in stack] == [_A_ROUTE.sub("", r) for r in chain], (case, stack, chain)
        for a, b in zip(stack, chain):
            assert a == b or (a.endswith(" a=tma") and b.endswith(" a=gather")), (case, a, b)
        fwd = [r for r in stack if r.startswith("fwd ")]
        bwd = [r for r in stack if r.startswith("bwd ")]
        inner_fwd.update(fwd[1:])      # forward: layer 0 first
        inner_bwd.update(bwd[:-1])     # backward: the top layer first, layer 0 last
        k2048 |= any(re.search(r"forward x-projection: M=\d+ N=\d+ K=2048 math=3xtf32", r) for r in stack)
    missing_f = set(FWD_LINE.values()) - inner_fwd
    missing_b = set(BWD_LINE.values()) - inner_bwd
    assert not missing_f and not missing_b, (sorted(missing_f), sorted(missing_b))
    assert k2048, "no tensor-core x-projection with K = 2048 ran"


# ---- 2. against float64 -----------------------------------------------------------------------------------------------

def _f64_run(layers, dt, x, lens, hx, masks, wy, ws):
    from torch.nn.utils.rnn import pack_padded_sequence  # noqa: F401  (oracle.stacked packs)

    mods = [m.to(dt) for m in layers]
    for m in mods:
        m.zero_grad(set_to_none=True)
    xx = x.to(dt).clone().requires_grad_(True)
    st = [s.to(dt).clone().requires_grad_(True) for s in hx]
    y, sts = chained(mods, xx, lens, tuple(st) if len(st) == 2 else st[0],
                     None if masks is None else [mk.to(dt) for mk in masks])
    loss = (y * wy.to(dt)).sum() + sum((s * w.to(dt)).sum() for s, w in zip(sts, ws))
    loss.backward()
    res = {"y": y, **dict(zip(("h_n", "c_n"), sts)), "dx": xx.grad}
    for l, m in enumerate(mods):
        res.update({"d" + n.replace("_l0", f"_l{l}"): q.grad for n, q in m.named_parameters()})
    res.update(dict(zip(("dh_0", "dc_0"), (s.grad for s in st))))
    return {k: v.detach().double().numpy() for k, v in res.items()}


def _mine_run(ref, mode, x, lens, hx, wy, ws, p):
    import b200rnn
    from b200rnn.functional import rnn_forward

    mine = b200rnn.from_torch(ref).to(DEV).train(p > 0)
    xx = x.to(DEV).requires_grad_(True)
    st = [s.to(DEV).requires_grad_(True) for s in hx]
    rng = torch.tensor((SEED, OFFSET), dtype=torch.int64, device=DEV)
    out = rnn_forward(xx, mine._flat_weights, _cfg(mine, mode == "tf32"), rng, lengths=lens,
                      hx=tuple(st) if len(st) == 2 else st[0])
    y, states = out[0], out[1:]
    loss = (y * wy.to(DEV)).sum() + sum((s * w.to(DEV)).sum() for s, w in zip(states, ws))
    loss.backward()
    res = {"y": y, **dict(zip(("h_n", "c_n"), states)), "dx": xx.grad}
    res.update({"d" + n: q.grad for n, q in mine.named_parameters()})
    res.update(dict(zip(("dh_0", "dc_0"), (s.grad for s in st))))
    return {k: v.detach().cpu().double().numpy() for k, v in res.items()}


def _free_running(name, regime, L, p=0.3, T=24):
    kind, I, H, B, bi, P, mode = CONFIGS[name]
    if regime == "large_input":
        I = 1024
    D, HO = (2 if bi else 1), (P or H)
    ref = _stack_model(kind, I, H, L, bi, P, regime, dropout=p)
    x = _input("default" if regime == "radius" else regime, T, B, I)
    lens = _ragged_lengths(B, T)
    lens[1 % B] = 1
    g = torch.Generator().manual_seed(4)
    hx = [0.5 * torch.randn(L * D, B, HO, generator=g)] + (
        [0.5 * torch.randn(L * D, B, H, generator=g)] if kind == "lstm" else [])
    wy = torch.randn(T, B, D * HO, generator=g) * (torch.arange(T)[:, None] < lens[None, :]).float()[:, :, None]
    ws = [torch.randn(s.shape, generator=g) for s in hx]
    n = T * B * D * HO
    masks = [torch.from_numpy(philox.dropout_factor(SEED, OFFSET, l, n, p).reshape(T, B, D * HO))
             for l in range(L - 1)] if p > 0 else None
    layers = split_layers(ref)
    r64 = _f64_run(layers, torch.float64, x, lens, hx, masks, wy, ws)
    r32 = _f64_run(layers, torch.float32, x, lens, hx, masks, wy, ws)
    got = _mine_run(ref, mode, x, lens, hx, wy, ws, p)
    assert sorted(got) == sorted(r64)
    if kind == "rnn_relu":   # the precondition of the bound: one branch at every top-layer pre-activation
        for r in (got, r32):
            assert np.array_equal(r["y"] > 0, r64["y"] > 0), (name, regime, "a relu branch differs from float64")
    scale = 2.0 ** 13 if mode == "tf32" else 1.0
    bad = []
    for k, want in r64.items():
        e_k, e_t = _norm_err(got[k], want), _norm_err(r32[k], want)
        _record_ratio("free_running_err_over_torch32", f"{name}_L{L}", regime, k, e_k / max(e_t, 1e-300))
        if not e_k <= 4 * scale * e_t + 1e-6:
            bad.append((k, e_k, e_t))
    return bad


# the relu RNN stays at L = 2: at L = 3 its branch precondition (every top-layer pre-activation on float64's side of
# 0 in the kernel and in stock fp32) failed in the default regime
FREE_L3 = ["gru256_tc8_3xtf32", "bilstm128_wide", "bilstmp_h256_p128", "gru_h1024_bi", "tanh_h1008_bi"]


@pytest.mark.parametrize("regime", ["default", "stress", "large_input"])
@pytest.mark.parametrize("name,L", [(n, 2) for n in CONFIGS] + [(n, 3) for n in FREE_L3])
def test_free_running_stack_vs_f64(name, L, regime):
    """ragged, hx, dropout 0.3; regime `stress`: saturated, or radius for the relu RNN"""
    if regime == "stress":
        regime = "radius" if CONFIGS[name][0] == "rnn_relu" else "saturated"
    bad = _free_running(name, regime, L)
    assert not bad, (name, L, regime, bad)


# per-step on the inner layer: the chain's layer 1 with the kernel's own dropped layer-0 output as x
PER_STEP = ["gru_h1024_bi", "lstm_h1008_bi", "gru256_bs4", "gru128", "bilstm256", "bilstm128", "bilstmp_h128_p64"]


@pytest.mark.parametrize("regime", ["default", "saturated"])
@pytest.mark.parametrize("name", PER_STEP)
def test_inner_layer_per_step_within_rounding_bound(name, regime):
    import b200rnn
    from b200rnn.functional import rnn_forward
    from oracle.rnn_numpy import gru_step, lstm_step

    kind, I, H, B, bi, P, mode = CONFIGS[name]
    T, D, HO, p = 24, (2 if bi else 1), (P or H), 0.3
    K = D * HO
    ref = _stack_model(kind, I, H, 2, bi, P, regime, dropout=p)
    l0, l1 = [b200rnn.from_torch(m).to(DEV) for m in split_layers(ref)]
    x = _input("saturated" if regime == "saturated" else "default", T, B, I)
    g = torch.Generator().manual_seed(6)
    hx = [0.5 * torch.randn(D, B, HO, generator=g)] + ([0.5 * torch.randn(D, B, H, generator=g)] if kind == "lstm" else [])
    with torch.no_grad():
        y0 = rnn_forward(x.to(DEV), l0._flat_weights, _cfg(l0, False))[0]
        keep, scale = _drop_args(T, B, K, p, 0, (SEED, OFFSET))
        x1 = _dropped(y0, keep, scale)
    x64 = x1.cpu().double().numpy()
    ws = []
    for d in range(D):
        sfx = "_l0" + ("_reverse" if d else "")
        names = ("weight_ih", "weight_hh", "bias_ih", "bias_hh") + (("weight_hr",) if P else ())
        ws.append([getattr(l1, n + sfx).detach().cpu().double().numpy() for n in names])
    bound = kappa(K) * U32
    worst = 0.0
    if kind == "gru":   # one call: the trajectory is y itself; the reverse half's previous state is y[t + 1]
        with torch.no_grad():
            y = rnn_forward(x1, l1._flat_weights, _cfg(l1, False), hx=hx[0].to(DEV))[0].cpu().double().numpy()
        h0 = hx[0].double().numpy()
        for d in range(D):
            yd = y[:, :, d * H:(d + 1) * H]
            for t in range(T):
                tp = t + 1 if d else t - 1
                h_prev = yd[tp] if 0 <= tp < T else h0[d]
                h64, S = gru_step(x64[t], h_prev, *ws[d])
                worst = max(worst, (np.abs(yd[t] - h64) / (bound * S)).max())
    else:   # chained one-step calls through (h, c), which return the cell state as well
        h, c = (s.to(DEV) for s in hx)
        xs = x1.cpu()
        for t in range(T):
            with torch.no_grad():
                _, h1, c1 = rnn_forward(xs[t:t + 1].to(DEV), l1._flat_weights, _cfg(l1, False), hx=(h, c))
            hp, cp, hn, cn = (a.cpu().double().numpy() for a in (h, c, h1, c1))
            for d in range(D):
                h64, c64, S_h, S_c = lstm_step(x64[t], hp[d], cp[d], *ws[d])
                for got, want, S in ((hn[d], h64, S_h), (cn[d], c64, S_c)):
                    worst = max(worst, (np.abs(got - want) / (bound * S)).max())
            h, c = h1, c1
    _record_ratio("inner_per_step_max_err_over_bound", f"{name}_K{K}", regime, "T%d" % T, worst)
    assert worst <= 1.0, (name, regime, K, worst)
