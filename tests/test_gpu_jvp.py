"""Forward-mode AD through the sequence modules on the GPU: torch.func.jvp / jacfwd and eager forward_ad dual tensors
against stock torch in float64 on the CPU, the primal left untouched, dropout, the adjoint identity with the backward,
one tangent recurrence launch per layer for M directions, and the refusals."""
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.autograd.forward_ad as fwAD
from torch import nn
from torch.func import functional_call, jacfwd, jvp, vjp

import b200rnn
from b200rnn import _lib
from oracle import philox

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOUND = 1e-4   # max error relative to each tensor's largest entry, the gradients' bound elsewhere in the suite


def _modules(kind, H, L, D, I=24, batch_first=False, dropout=0.0, seed=0):
    torch.manual_seed(seed)
    if kind.startswith("rnn"):
        ref = nn.RNN(I, H, num_layers=L, bidirectional=D == 2, batch_first=batch_first, dropout=dropout,
                     nonlinearity=kind.split("_")[1])
    else:
        cls = nn.GRU if kind == "gru" else nn.LSTM
        ref = cls(I, H, num_layers=L, bidirectional=D == 2, batch_first=batch_first, dropout=dropout)
    with torch.no_grad():   # away from default init: weights large enough that the gates saturate somewhere
        for p in ref.parameters():
            p.mul_(2.0)
    mine = b200rnn.from_torch(copy.deepcopy(ref)).to(DEV)
    return ref.double(), mine


def _fn(module, with_hx):
    def f(params, x, *hx):
        y, h = functional_call(module, params, (x, hx[0] if with_hx else None))
        return (y, *h) if isinstance(h, tuple) else (y, h)
    return f


def _inputs(kind, H, L, D, B, T, I, batch_first, unbatched, with_hx, gen):
    shape = (T, I) if unbatched else ((B, T, I) if batch_first else (T, B, I))
    x = torch.randn(shape, generator=gen, dtype=torch.float64)
    sshape = (L * D, H) if unbatched else (L * D, B, H)
    hx = ()
    if with_hx:
        h0 = 0.5 * torch.randn(sshape, generator=gen, dtype=torch.float64)
        hx = ((h0, 0.5 * torch.randn(sshape, generator=gen, dtype=torch.float64)) if kind == "lstm" else h0,)
    return x, hx


def _rand_like(tree, gen):
    return torch.utils._pytree.tree_map(
        lambda t: torch.randn(t.shape, generator=gen, dtype=torch.float64).to(t.dtype).to(t.device), tree)


def _to_dev(tree):
    return torch.utils._pytree.tree_map(lambda t: t.float().to(DEV), tree)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# (kind, H, L, D, B, T, batch_first, unbatched, hx): every mode, hidden size 16 .. 1024 (1024: the L2 tier), both
# directions, 1-3 layers, batch_first, unbatched input, with and without hx, B from 1 to 200 (several waves), T 1 and 120
CASES = [
    ("gru", 16, 1, 1, 1, 1, False, False, False),
    ("gru", 48, 2, 2, 5, 30, True, False, True),
    ("gru", 128, 2, 1, 64, 120, True, False, False),
    ("gru", 256, 2, 2, 200, 120, False, False, True),
    ("gru", 320, 3, 1, 9, 20, False, False, True),
    ("gru", 1024, 1, 2, 4, 12, False, False, True),
    ("lstm", 16, 1, 2, 1, 120, False, True, True),
    ("lstm", 128, 2, 2, 64, 30, False, False, True),
    ("lstm", 256, 1, 1, 33, 1, True, False, True),
    ("lstm", 512, 1, 1, 16, 120, False, False, False),
    ("lstm", 1024, 2, 1, 3, 10, True, False, True),
    ("rnn_tanh", 48, 3, 2, 200, 25, True, False, True),
    ("rnn_tanh", 256, 2, 1, 64, 120, False, False, False),
    ("rnn_tanh", 512, 1, 2, 2, 40, False, True, True),
    ("rnn_relu", 128, 2, 2, 100, 50, False, False, True),
    ("rnn_relu", 320, 1, 1, 7, 1, False, False, False),
    ("rnn_relu", 1024, 1, 1, 5, 16, True, False, True),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(map(str, c)))
def test_jvp_against_float64(case):
    kind, H, L, D, B, T, bf, unb, with_hx = case
    I = 24
    ref, mine = _modules(kind, H, L, D, I, bf)
    ref.eval(), mine.eval()
    gen = torch.Generator().manual_seed(1)
    x, hx = _inputs(kind, H, L, D, B, T, I, bf, unb, with_hx, gen)
    p64 = {n: p.detach() for n, p in ref.named_parameters()}
    tp, tx, thx = _rand_like(p64, gen), _rand_like(x, gen), _rand_like(hx, gen)
    want_p, want_t = jvp(_fn(ref, with_hx), (p64, x, *hx), (tp, tx, *thx))
    p32 = {n: p.detach() for n, p in mine.named_parameters()}
    assert set(p32) == set(p64)
    got_p, got_t = jvp(_fn(mine, with_hx), (p32, _to_dev(x), *_to_dev(hx)), (_to_dev(tp), _to_dev(tx), *_to_dev(thx)))
    for g, w in zip(got_t, want_t):
        assert g.shape == w.shape
        assert _rel(g, w) <= BOUND, (_rel(g, w), case)
    for g, w in zip(got_p, want_p):
        assert _rel(g, w) <= BOUND


def _dual_call(mine, p32, x, hx, tp, tx, thx):
    with fwAD.dual_level():
        pd = {n: fwAD.make_dual(p, tp[n]) for n, p in p32.items()}
        xd = fwAD.make_dual(x, tx)
        hd = torch.utils._pytree.tree_map(fwAD.make_dual, hx, thx) if hx is not None else None
        out = functional_call(mine, pd, (xd, hd))
        flat = (out[0], *out[1]) if isinstance(out[1], tuple) else out
        return [fwAD.unpack_dual(o).primal.clone() for o in flat], [fwAD.unpack_dual(o).tangent.clone() for o in flat]


@pytest.mark.parametrize("kind", ["gru", "lstm", "rnn_tanh"])
def test_eager_dual_tensors_equal_torch_func_jvp_bitwise(kind):
    ref, mine = _modules(kind, 48, 2, 2)
    mine.eval()
    gen = torch.Generator().manual_seed(2)
    x, hx = _inputs(kind, 48, 2, 2, 6, 17, 24, False, False, True, gen)
    p32 = {n: p.detach() for n, p in mine.named_parameters()}
    tp, tx, thx = _to_dev(_rand_like(p32, gen)), _to_dev(_rand_like(x, gen)), _to_dev(_rand_like(hx, gen))
    x, hx = _to_dev(x), _to_dev(hx)
    _, want = jvp(_fn(mine, True), (p32, x, *hx), (tp, tx, *thx))
    _, got = _dual_call(mine, p32, x, hx[0], tp, tx, thx[0])
    for g, w in zip(got, want):
        assert torch.equal(g, w)


@pytest.mark.parametrize("kind", ["gru", "lstm", "rnn_relu"])
def test_primal_of_jvp_is_the_plain_forward_bitwise_with_dropout(kind):
    _, mine = _modules(kind, 128, 3, 2, dropout=0.3)
    mine.train()
    x = torch.randn(20, 8, 24, device=DEV)
    rng = mine._rng_state.clone()
    with torch.no_grad():
        plain = mine(x)
    plain = (plain[0], *plain[1]) if isinstance(plain[1], tuple) else plain
    mine._rng_state.copy_(rng)
    p32 = {n: p.detach() for n, p in mine.named_parameters()}
    primal, _ = jvp(_fn(mine, False), (p32, x), (_rand_like(p32, torch.Generator()), torch.randn_like(x)))
    for a, b in zip(primal, plain):
        assert torch.equal(a, b)
    assert not torch.equal(mine._rng_state, rng)   # the jvp's forward drew its mask as a plain call does


def _layer_stack(ref, kind, L, D, I, H):
    """one single-layer float64 stock module per layer of `ref`, with its weights"""
    layers = []
    for l in range(L):
        Il = I if l == 0 else D * H
        if kind.startswith("rnn"):
            m = nn.RNN(Il, H, bidirectional=D == 2, nonlinearity=kind.split("_")[1])
        else:
            m = (nn.GRU if kind == "gru" else nn.LSTM)(Il, H, bidirectional=D == 2)
        m = m.double()
        with torch.no_grad():
            for n, p in m.named_parameters():
                p.copy_(getattr(ref, n.replace("_l0", f"_l{l}")))
        layers.append(m)
    return layers


@pytest.mark.parametrize("kind", ["gru", "lstm", "rnn_tanh"])
def test_dropout_tangent_against_float64_with_the_philox_masks(kind):
    """train mode with inter-layer dropout: the tangent against stock float64 jvp through the layers, with the masks the
    kernels draw (oracle/philox.py, keyed by the module's rng state at the call)"""
    L, D, H, T, B, I, p = 3, 2, 64, 15, 6, 24, 0.4
    ref, mine = _modules(kind, H, L, D, I, dropout=p)
    mine.train()
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(T, B, I, generator=gen, dtype=torch.float64)
    v = torch.randn(T, B, I, generator=gen, dtype=torch.float64)
    seed, off = (int(t) & (2 ** 64 - 1) for t in mine._rng_state.tolist())
    p32 = {n: p.detach() for n, p in mine.named_parameters()}
    _, ydot = jvp(lambda x: functional_call(mine, p32, (x,))[0], (_to_dev(x),), (_to_dev(v),))
    layers = _layer_stack(ref, kind, L, D, I, H)
    fac = [torch.from_numpy(philox.dropout_factor(seed, off, l, T * B * D * H, p)).double().view(T, B, D * H)
           for l in range(L - 1)]

    def f(h):
        for l, m in enumerate(layers):
            h = m(h)[0]
            if l < L - 1:
                h = h * fac[l]
        return h

    _, want = jvp(f, (x,), (v,))
    assert _rel(ydot, want) <= BOUND
    # the masks matter: without dropout the tangent differs
    mine.eval()
    _, y_eval = jvp(lambda x: functional_call(mine, p32, (x,))[0], (_to_dev(x),), (_to_dev(v),))
    assert _rel(y_eval, want) > 1e-2


# which inputs carry a tangent: each group alone, so that each GEMM of the tangent pre-activations is the writing one
# (x: W_ih x'; params: W_ih' x; hx: none, pre = 0 on layer 0; weight_hh: the zeroed buffer and the GRU's h side alone)
GROUPS = ["x", "params", "hx", "weight_hh"]


@pytest.mark.parametrize("group", GROUPS)
@pytest.mark.parametrize("kind", ["gru", "lstm", "rnn_relu"])
def test_jvp_of_one_input_group_against_float64(kind, group):
    H, L, D, B, T, I = 48, 2, 2, 7, 20, 24
    ref, mine = _modules(kind, H, L, D, I)
    ref.eval(), mine.eval()
    gen = torch.Generator().manual_seed(4)
    x, hx = _inputs(kind, H, L, D, B, T, I, False, False, True, gen)

    def run(module, params, x, hx, to):
        f = _fn(module, True)
        if group == "x":
            return jvp(lambda x: f(params, x, *hx), (x,), (to(_rand_like(x, gen)),))[1]
        if group == "hx":
            return jvp(lambda *h: f(params, x, *h), hx, to(_rand_like(hx, gen)))[1]
        sub = {n: p for n, p in params.items() if group == "params" or "weight_hh" in n}
        return jvp(lambda s: f({**params, **s}, x, *hx), (sub,), (to(_rand_like(sub, gen)),))[1]

    p64 = {n: p.detach() for n, p in ref.named_parameters()}
    gen.manual_seed(5)
    want = run(ref, p64, x, hx, lambda t: t)
    gen.manual_seed(5)
    p32 = {n: p.detach() for n, p in mine.named_parameters()}
    got = run(mine, p32, _to_dev(x), _to_dev(hx), _to_dev)
    for g, w in zip(got, want):
        assert _rel(g, w) <= BOUND, (_rel(g, w), kind, group)


@pytest.mark.parametrize("dual", ["x", "weight"])
def test_create_graph_gradient_inside_a_dual_level_is_refused(dual):
    """forward-over-reverse with a plain output gradient: the saved input carries the tangent, dy does not"""
    gru = b200rnn.from_torch(nn.GRU(16, 32)).to(DEV)
    x = torch.randn(5, 3, 16, device=DEV, requires_grad=True)
    params = {n: p.detach() for n, p in gru.named_parameters()}
    with fwAD.dual_level():
        if dual == "x":
            y = functional_call(gru, params, (fwAD.make_dual(x, torch.ones_like(x)),))[0]
        else:
            w = params["weight_ih_l0"]
            y = functional_call(gru, {**params, "weight_ih_l0": fwAD.make_dual(w, torch.ones_like(w))}, (x,))[0]
        with pytest.raises(_lib.B200RNNError, match="forward-over-reverse"):
            torch.autograd.grad(y.sum() + (x ** 2).sum(), x, create_graph=True)


@pytest.mark.parametrize("kind", ["gru", "lstm", "rnn_tanh"])
def test_adjoint_identity_with_the_backward(kind):
    _, mine = _modules(kind, 256, 2, 2)
    mine.eval()
    x = torch.randn(40, 16, 24, device=DEV)
    v = torch.randn_like(x)
    p32 = {n: p.detach() for n, p in mine.named_parameters()}
    f = lambda x: functional_call(mine, p32, (x,))[0]  # noqa: E731
    y, jv = jvp(f, (x,), (v,))
    u = torch.randn_like(y)
    _, pullback = vjp(f, x)
    (jtu,) = pullback(u)
    a, b = float((u.double() * jv.double()).sum()), float((jtu.double() * v.double()).sum())
    assert abs(a - b) <= 1e-4 * max(abs(a), abs(b), 1.0)


def test_jacfwd_over_x_equals_stock_float64_and_chunked_directions_agree():
    ref, mine = _modules("lstm", 16, 2, 2, I=5)
    ref.eval(), mine.eval()
    x = torch.randn(4, 3, 5, dtype=torch.float64)
    want = jacfwd(lambda x: ref(x)[0])(x)
    f = lambda x: mine(x)[0]  # noqa: E731
    got = jacfwd(f)(x.float().to(DEV))
    assert got.shape == want.shape
    assert _rel(got, want) <= BOUND
    # the directions in chunks of 7 (calls of 7 and fewer directions) compute what one call of all 60 does
    xd = x.float().to(DEV)
    basis = torch.eye(xd.numel(), device=DEV).view(xd.numel(), *xd.shape)
    cols = lambda **kw: torch.vmap(lambda t: jvp(f, (xd,), (t,))[1], **kw)(basis)  # noqa: E731
    assert torch.equal(cols(chunk_size=7), cols())
    assert torch.equal(cols().movedim(0, -1).reshape(got.shape), got)


def test_jacfwd_runs_one_tangent_launch_per_layer():
    script = (
        "import torch, b200rnn\n"
        "from torch import nn\n"
        "torch.manual_seed(0)\n"
        "m = b200rnn.from_torch(nn.GRU(8, 48, num_layers=3, bidirectional=True)).cuda().eval()\n"
        "x = torch.randn(5, 4, 8, device='cuda')\n"
        "torch.func.jacfwd(lambda x: m(x)[0])(x)\n"
        "torch.cuda.synchronize()\n")
    env = dict(os.environ, B200RNN_DEBUG="1", PYTHONPATH=os.path.join(ROOT, "icassp2022-depression_b200"))
    out = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stderr.splitlines() if "[b200rnn] tan " in ln]
    assert len(lines) == 3, lines   # one launch per layer for all 5 * 4 * 8 = 160 directions
    # 160 directions x 2 directions of the layer x the batch slices
    assert all(int(ln.split("need ")[1].split()[0]) % 320 == 0 for ln in lines), lines


def test_refusals():
    x = torch.randn(5, 4, 32, device=DEV)
    lstm_p = b200rnn.from_torch(nn.LSTM(32, 128, proj_size=32)).to(DEV)
    gru = b200rnn.from_torch(nn.GRU(32, 64)).to(DEV)
    f = lambda m: (lambda x: m(x)[0])  # noqa: E731
    with pytest.raises(_lib.B200RNNError, match="proj_size"):
        jvp(f(lstm_p), (x,), (x,))
    with fwAD.dual_level(), pytest.raises(_lib.B200RNNError, match="proj_size"):
        lstm_p(fwAD.make_dual(x, x))
    g16 = copy.deepcopy(gru).half()
    with fwAD.dual_level(), pytest.raises(_lib.B200RNNError, match="float32"):
        g16(fwAD.make_dual(x.half(), x.half()))
    with pytest.raises(_lib.B200RNNError):
        jvp(f(g16), (x.half(),), (x.half(),))
    with torch.autocast("cuda"), fwAD.dual_level(), pytest.raises(_lib.B200RNNError, match="autocast"):
        gru(fwAD.make_dual(x, x))
    loss = lambda x: gru(x)[0].square().sum()  # noqa: E731
    with pytest.raises(_lib.B200RNNError, match="forward-over-reverse"):
        torch.func.hessian(loss)(torch.randn(2, 1, 32, device=DEV))
    with pytest.raises(_lib.B200RNNError, match="forward-over-reverse"):
        jvp(torch.func.grad(loss), (x,), (x,))
    with pytest.raises(_lib.B200RNNError, match="reverse-over-forward"):
        torch.func.grad(lambda x: jvp(f(gru), (x,), (x,))[1].sum())(x)
