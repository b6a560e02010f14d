"""16-bit GRU / LSTM / RNN modules on the GPU against a float64 oracle.

The oracle restates the 16-bit problem in float64: the same rounded input and weights, every layer run by stock torch
in float64, and each inner layer's output rounded to the dtype before the next layer reads it (straight through in the
backward), as the library and stock torch materialise it. Bounds: an output is within half a dtype ulp of its value
plus 2e-5 (the fp32 recurrence before the one rounding), plus one ulp of the largest output with more than one layer
(an inner rounding that falls the other way); a gradient within one dtype ulp of its largest element plus
1e-4 of that element. Stock cuDNN in the same dtype is measured against the same oracle and printed beside ours.
"""
import math
import re

import pytest
import torch

import b200rnn

pytestmark = pytest.mark.gpu

DT = {"f16": torch.float16, "bf16": torch.bfloat16}
MANT = {torch.float16: 10, torch.bfloat16: 7}
STOCK = {"gru": torch.nn.GRU, "lstm": torch.nn.LSTM, "tanh": torch.nn.RNN, "relu": torch.nn.RNN}
MINE = {"gru": b200rnn.GRU, "lstm": b200rnn.LSTM, "tanh": b200rnn.RNN, "relu": b200rnn.RNN}


def _kw(kind):
    return {"nonlinearity": kind} if kind in ("tanh", "relu") else {}


def _ulp(v, dt):
    return 2.0 ** (math.floor(math.log2(max(abs(v), 2.0 ** -14))) - MANT[dt])


def _oracle(mod, x, hx, dt, masks=None):
    """float64 forward and gradients of the 16-bit problem (CPU), layer by layer with the rounding between layers;
    masks[l] (optional): the inter-layer dropout factor (0 or 1 / (1 - p)) of layer l's output, applied between the two
    roundings"""
    L, D = mod.num_layers, 2 if mod.bidirectional else 1
    lstm = isinstance(mod, b200rnn.LSTM)
    xin = x.detach().double().cpu().requires_grad_(True)
    h0 = None
    if hx is not None:
        h0 = tuple(s.detach().double().cpu().requires_grad_(True) for s in (hx if lstm else (hx,)))
    params, inp, hs, cs = [], xin, [], []
    for layer in range(L):
        ref = STOCK[mod._kind](inp.size(-1), mod.hidden_size, num_layers=1, bidirectional=mod.bidirectional,
                               batch_first=mod.batch_first, dtype=torch.float64, **_kw(mod._kind))
        with torch.no_grad():
            for name, p in ref.named_parameters():
                base, rev = name.split("_l0")
                p.copy_(getattr(mod, f"{base}_l{layer}{rev}").detach().double().cpu())
        params += list(ref.parameters())
        st = None
        if h0 is not None:
            st = tuple(s[layer * D:(layer + 1) * D] for s in h0)
            st = st if lstm else st[0]
        out, hn = ref(inp, st)
        hs.append(hn[0] if lstm else hn)
        if lstm:
            cs.append(hn[1])
        if layer + 1 < L:
            r = out.to(dt).double()
            if masks is not None:
                m = masks[layer].double().cpu()
                inp = out * m + ((r * m).to(dt).double() - out * m).detach()
            else:
                inp = out + (r - out).detach()
        else:
            inp = out
    h_n = torch.cat(hs)
    res = (inp, h_n, torch.cat(cs)) if lstm else (inp, h_n)
    return res, xin, h0, params


def _masks(mod, T, B, p):
    """the dropout factors the next forward of `mod` draws for each inner layer: the library's Philox stream l keyed by
    the module's device RNG state, regenerated through b200rnn_debug_dropout on a tensor of ones"""
    import ctypes
    from b200rnn import _lib
    lib = _lib.load()
    lib.b200rnn_debug_dropout.restype = ctypes.c_int
    lib.b200rnn_debug_dropout.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_float,
                                          ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p,
                                          ctypes.c_void_p]
    seed, off = (int(v) for v in mod._rng_state.tolist())
    D = 2 if mod.bidirectional else 1
    n = T * B * D * mod.hidden_size
    ones = torch.ones(n, device="cuda")
    hdr = torch.zeros(2, dtype=torch.int64, device="cuda")
    out = []
    for layer in range(mod.num_layers - 1):
        m = torch.empty_like(ones)
        _lib.check(lib.b200rnn_debug_dropout(ones.data_ptr(), m.data_ptr(), n, p, seed, off, layer, hdr.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream), "debug_dropout")
        out.append(m.view(T, B, D * mod.hidden_size))
    torch.cuda.synchronize()
    return out


def _run(kind, dt, H, L=1, bi=False, batch_first=False, T=20, B=8, I=64, hx=False, seed=0, p=0.0):
    torch.manual_seed(seed)
    mod = MINE[kind](I, H, num_layers=L, bidirectional=bi, batch_first=batch_first, dropout=p, dtype=dt,
                     **_kw(kind)).cuda()
    mod._kind = kind
    masks = _masks(mod, T, B, p) if p > 0 else None
    shape = (B, T, I) if batch_first else (T, B, I)
    x = torch.randn(shape, device="cuda").to(dt).requires_grad_(True)
    D = 2 if bi else 1
    state = None
    if hx:
        s = [(0.5 * torch.randn(L * D, B, H, device="cuda")).to(dt).requires_grad_(True)
             for _ in range(2 if kind == "lstm" else 1)]
        state = tuple(s) if kind == "lstm" else s[0]
    out = mod(x, state)
    y, fin = out[0], out[1]
    finals = list(fin) if kind == "lstm" else [fin]
    assert y.dtype == dt and all(f.dtype == dt for f in finals)
    w = torch.randn_like(y, dtype=torch.float32).to(dt)
    loss = (y.float() * w.float()).sum() + sum(f.float().sum() for f in finals)
    loss.backward()
    ref, xin, h0, params = _oracle(mod, x, state, dt, masks)
    rloss = (ref[0] * w.double().cpu()).sum() + sum(r.sum() for r in ref[1:])
    rloss.backward()
    # outputs. Above layer 0 an inner output that rounds the other way than the oracle's moves the next layer's input
    # by one ulp: one ulp of the largest output is allowed on top
    for got, want in zip([y] + finals, ref):
        g, r = got.double().cpu(), want.detach()
        flip = _ulp(r.abs().max().item(), dt) if L > 1 else 0.0
        bound = torch.tensor([0.5 * _ulp(v, dt) for v in r.flatten().tolist()]).view_as(r) + 2e-5 + flip
        assert ((g - r).abs() <= bound).all(), (kind, dt, H, (g - r).abs().max().item())
    # gradients
    pairs = [(x.grad, xin.grad)] + [(p.grad, q.grad) for p, q in zip(mod.parameters(), params)]
    if h0 is not None:
        pairs += [(s.grad, r.grad) for s, r in zip(state if kind == "lstm" else (state,), h0)]
    for got, want in pairs:
        assert got is not None and got.dtype == dt
        m = want.abs().max().item()
        err = (got.double().cpu() - want).abs().max().item()
        assert err <= _ulp(m, dt) + 1e-4 * m, (kind, dt, H, err, m)
    return mod, x, state, ref, masks


@pytest.mark.parametrize("dtn", ["f16", "bf16"])
@pytest.mark.parametrize("kind", ["gru", "lstm", "tanh", "relu"])
@pytest.mark.parametrize("H", [64, 128, 256, 512, 1024])
def test_forward_backward_against_float64(kind, dtn, H):
    _run(kind, DT[dtn], H, T=12 if H >= 512 else 20, B=8)


@pytest.mark.parametrize("dtn", ["f16", "bf16"])
@pytest.mark.parametrize("kind,H", [("gru", 256), ("lstm", 128), ("lstm", 640), ("lstm", 656), ("gru", 752), ("gru", 768), ("tanh", 96)])
def test_two_layers_bidirectional_batch_first_hx(kind, dtn, H):
    _run(kind, DT[dtn], H, L=2, bi=True, batch_first=True, hx=True, T=16, B=5, I=40)


def test_long_and_several_waves_of_clusters():
    _run("gru", torch.float16, 256, T=120, B=128, I=256)
    _run("lstm", torch.bfloat16, 384, T=30, B=300, I=128, L=2)


@pytest.mark.parametrize("dtn", ["f16", "bf16"])
@pytest.mark.parametrize("kind,H", [("gru", 256), ("lstm", 640), ("relu", 96)])
def test_dropout_in_train_mode_against_float64(kind, dtn, H):
    """the round - dropout - round chain between layers, forward and backward, with the mask the library draws"""
    p = 0.3
    _, _, _, _, masks = _run(kind, DT[dtn], H, L=3, T=12, B=16, I=64, p=p)
    keep = torch.cat([(m != 0).float().flatten() for m in masks]).mean().item()
    n = sum(m.numel() for m in masks)
    assert abs(keep - (1 - p)) < 5 * math.sqrt(p * (1 - p) / n), keep


@pytest.mark.parametrize("dtn", ["f16", "bf16"])
@pytest.mark.parametrize("kind,H", [("lstm", 128), ("gru", 720), ("tanh", 64)])
def test_packed_sequence_against_float64(kind, dtn, H):
    """ragged PackedSequence, forward and backward: each sequence's rows against the oracle run on that sequence alone
    (the parameter gradients are the sums over the sequences)"""
    dt = DT[dtn]
    torch.manual_seed(3)
    mod = MINE[kind](32, H, num_layers=2, bidirectional=True, dtype=dt, **_kw(kind)).cuda()
    mod._kind = kind
    lens = [9, 4, 7, 1, 9]
    x = torch.randn(9, 5, 32, device="cuda").to(dt).requires_grad_(True)
    packed = torch.nn.utils.rnn.pack_padded_sequence(x, torch.tensor(lens), enforce_sorted=False)
    out = mod(packed)
    finals = list(out[1]) if kind == "lstm" else [out[1]]
    assert out[0].data.dtype == dt and all(f.dtype == dt for f in finals)
    ypad, _ = torch.nn.utils.rnn.pad_packed_sequence(out[0])
    w = torch.randn_like(ypad, dtype=torch.float32).to(dt)
    ((ypad.float() * w.float()).sum() + sum(f.float().sum() for f in finals)).backward()
    pgrads = None
    flip = lambda r: _ulp(r.abs().max().item(), dt)  # noqa: E731  two layers: one inner rounding may differ
    for b, n in enumerate(lens):
        ref, xin, _, params = _oracle(mod, x[:n, b:b + 1], None, dt)
        ((ref[0] * w[:n, b:b + 1].double().cpu()).sum() + sum(r.sum() for r in ref[1:])).backward()
        got = [ypad[:n, b:b + 1]] + [f[:, b:b + 1] for f in finals]
        for g, r in zip(got, ref):
            r = r.detach()
            bound = torch.tensor([0.5 * _ulp(v, dt) for v in r.flatten().tolist()]).view_as(r) + 2e-5 + flip(r)
            assert ((g.double().cpu() - r).abs() <= bound).all(), (kind, b, (g.double().cpu() - r).abs().max().item())
        assert (ypad[n:, b] == 0).all()
        gx, rx = x.grad[:n, b].double().cpu(), xin.grad[:, 0]
        m = rx.abs().max().item()
        assert (gx - rx).abs().max().item() <= _ulp(m, dt) + 1e-4 * m
        assert (x.grad[n:, b] == 0).all()
        pgrads = [q.grad.clone() for q in params] if pgrads is None else [a + q.grad for a, q in zip(pgrads, params)]
    for got, want in zip(mod.parameters(), pgrads):
        m = want.abs().max().item()
        err = (got.grad.double().cpu() - want).abs().max().item()
        assert err <= _ulp(m, dt) + 1e-4 * m, (kind, err, m)


@pytest.mark.parametrize("dtn", ["f16", "bf16"])
@pytest.mark.parametrize("kind,H", [("gru", 256), ("lstm", 1024), ("gru", 720)])
def test_error_no_larger_than_stock_cudnn(kind, H, dtn):
    """stock torch in the same dtype against the same oracle: our output error is no larger than cuDNN's"""
    dt = DT[dtn]
    mod, x, _, ref, _ = _run(kind, dt, H, T=30, B=16, I=64)
    stock = STOCK[kind](64, H, dtype=dt).cuda()
    stock.load_state_dict(mod.state_dict())
    with torch.no_grad():
        ys = stock(x)[0]
        ym = mod(x)[0]
    e_ours = (ym.double().cpu() - ref[0].detach()).abs().max().item()
    e_cudnn = (ys.double().cpu() - ref[0].detach()).abs().max().item()
    print(f"{kind}-{H} {dtn}: max |y - oracle| ours {e_ours:.3e}, cuDNN {e_cudnn:.3e}")
    assert e_ours <= e_cudnn, (e_ours, e_cudnn)


def test_deterministic_and_graph_replay():
    torch.manual_seed(1)
    mod = b200rnn.GRU(64, 720, num_layers=2, dtype=torch.bfloat16).cuda().eval()
    x = torch.randn(10, 16, 64, device="cuda").bfloat16()
    a, b = mod(x), mod(x)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    static_x = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        mod(static_x)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = mod(static_x)
    static_x.copy_(x)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], a[0]) and torch.equal(out[1], a[1])


def test_debug_lines_show_the_16bit_paths():
    import os
    import subprocess
    import sys
    code = ("import torch, b200rnn; m = b200rnn.LSTM(64, 640, dtype=torch.float16).cuda(); "
            "m(torch.randn(4, 8, 64, device='cuda').half())[0].float().sum().backward(); torch.cuda.synchronize()")
    pkg = os.path.dirname(os.path.dirname(os.path.abspath(b200rnn.__file__)))
    env = dict(os.environ, B200RNN_DEBUG="1", PYTHONPATH=pkg)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "math=f16 weights=native" in r.stderr, r.stderr
    assert "fwd anyh cfg LSTM VL=0 H=640" in r.stderr and "tier=smem w_hh=16bit" in r.stderr, r.stderr
    assert re.search(r"bwd anyh cfg LSTM VL=0 H=640 .*w_hh=16bit", r.stderr), r.stderr
