"""``torch.compile`` and ``torch.export`` of the b200rnn modules through the ``b200rnn::`` custom ops.

* ``torch.library.opcheck`` on every op over a small grid (16-bit dtypes and ``proj_size`` included).
* ``torch.compile(fullgraph=True)`` of the sequence modules and the cells: outputs and every gradient bitwise equal to
  eager. The compiled graph runs the same kernels in the same order, so equality is exact.
* The reference's model shells (``oracle.ref_models`` after ``install()``) in eval and in train mode with dropout,
  compiled with ``aot_eager`` so that the shell's own LayerNorm / Linear / softmax run torch's eager kernels as in the
  eager model (inductor would regenerate them with other roundings); the inter-layer dropout masks come from the same
  ``rng_state``, which checks that the op's mutation of it is carried.
* ``b200rnn.models`` with inductor: their shell fusions take the unfused expressions under compile, so they are
  compared within the parity bounds of ``test_gpu_models.py``.
* ``torch.export`` of the shells: the program calls ``b200rnn.rnn_forward``, matches eager bitwise and loads in a fresh
  process that only imports ``b200rnn``.
* ``mode="reduce-overhead"`` (CUDA-graph trees) replays a training step with dropout: each replay draws a new mask and
  equals the eager step from the same ``rng_state``.
"""
import os
import subprocess
import sys
import textwrap

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
# the forward ops return their workspace (reserve / saved) as an output, and its padding bytes are never written, so
# two calls differ there: opcheck's output comparisons through AOTAutograd run on the backward ops, and the forward's
# values through AOTAutograd are checked bitwise by the compile tests below
_FWD_OPCHECK = ("test_schema", "test_autograd_registration", "test_faketensor")


@pytest.fixture(autouse=True)
def _fresh_dynamo():
    torch._dynamo.reset()
    yield
    torch._dynamo.reset()


def _grads(params):
    return [p.grad.clone() if p.grad is not None else None for p in params]


def _zero(params):
    for p in params:
        p.grad = None


def _assert_same(a, b, what):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    assert a.dtype == b.dtype and a.shape == b.shape, what
    assert torch.equal(a, b), f"{what}: max |diff| {(a.float() - b.float()).abs().max().item():.3e}"


def _seq_module(kind, dtype=torch.float32, **kw):
    import b200rnn

    ctor = {"gru": b200rnn.GRU, "lstm": b200rnn.LSTM, "lstmp": b200rnn.LSTM, "tanh": b200rnn.RNN,
            "relu": b200rnn.RNN}[kind]
    if kind == "lstmp":
        kw["proj_size"] = 64
    if kind in ("tanh", "relu"):
        kw["nonlinearity"] = kind
    return ctor(48, 128, num_layers=2, bidirectional=True, batch_first=True, device=DEV, dtype=dtype, **kw)


# -- opcheck -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,dtype", [("gru", torch.float32), ("lstm", torch.float32), ("lstmp", torch.float32),
                                        ("tanh", torch.float32), ("gru", torch.float16), ("lstm", torch.bfloat16),
                                        ("relu", torch.float16)])
def test_opcheck_rnn_ops(kind, dtype):
    from b200rnn.ops import _rnn_attrs

    torch.manual_seed(0)
    m = _seq_module(kind, dtype)
    cfg = m._config()
    B, T = 3, 5
    x = torch.randn(B, T, 48, device=DEV, dtype=dtype, requires_grad=True).transpose(0, 1)
    HO = 64 if kind == "lstmp" else 128
    h_0 = torch.randn(4, B, HO, device=DEV, dtype=dtype, requires_grad=True)
    c_0 = torch.randn(4, B, 128, device=DEV, dtype=dtype) if kind.startswith("lstm") else None
    lengths = torch.tensor([5, 3, 4], dtype=torch.int32, device=DEV)
    rng = m._rng_state.clone()
    args = (x, m._flat_weights, h_0, c_0, lengths, rng, *_rnn_attrs(cfg), True)
    torch.library.opcheck(torch.ops.b200rnn.rnn_forward.default, args, test_utils=_FWD_OPCHECK)
    y, h_n, c_n, reserve = torch.ops.b200rnn.rnn_forward(*args)
    needs = [True, True, c_0 is not None] + [True] * len(m._flat_weights)
    bargs = (x.detach(), y.detach(), reserve, h_0.detach(), c_0, [w.detach() for w in m._flat_weights],
             torch.randn_like(y), torch.randn_like(h_n), torch.randn_like(c_n) if c_0 is not None else None, lengths,
             needs, *_rnn_attrs(cfg))
    torch.library.opcheck(torch.ops.b200rnn.rnn_backward.default, bargs)


@pytest.mark.parametrize("kind", ["gru", "lstm", "tanh"])
@pytest.mark.parametrize("bias", [True, False])
def test_opcheck_cell_ops(kind, bias):
    import b200rnn

    torch.manual_seed(0)
    cls = {"gru": b200rnn.GRUCell, "lstm": b200rnn.LSTMCell, "tanh": b200rnn.RNNCell}[kind]
    cell = cls(40, 48, bias=bias, device=DEV)
    weights = [cell.weight_ih, cell.weight_hh] + ([cell.bias_ih, cell.bias_hh] if bias else [])
    x = torch.randn(6, 40, device=DEV, requires_grad=True)
    h = torch.randn(6, 48, device=DEV, requires_grad=True)
    c = torch.randn(6, 48, device=DEV, requires_grad=True) if kind == "lstm" else None
    args = (x, h, c, weights, cell._mode, 40, 48, bias, False, True)
    torch.library.opcheck(torch.ops.b200rnn.cell_forward.default, args, test_utils=_FWD_OPCHECK)
    h_out, c_out, saved = torch.ops.b200rnn.cell_forward(*args)
    needs = [True, True, c is not None] + [True] * len(weights)
    bargs = (x.detach(), h.detach(), c.detach() if c is not None else None, saved, [w.detach() for w in weights],
             torch.randn_like(h_out), torch.randn_like(c_out) if c is not None else None, needs, cell._mode, 40, 48,
             bias, False)
    torch.library.opcheck(torch.ops.b200rnn.cell_backward.default, bargs)


# -- compile, modules ------------------------------------------------------------------------------------------------

def _run_seq(fn, m, x, hx):
    x = x.detach().clone().requires_grad_(True)
    hx = tuple(s.detach().clone().requires_grad_(True) for s in hx)
    _zero(m.parameters())
    y, state = fn(x, hx if len(hx) > 1 else hx[0])
    states = state if isinstance(state, tuple) else (state,)
    loss = (y.float() * torch.linspace(-1, 1, y.shape[-1], device=DEV)).sum() + sum(s.float().sum() for s in states)
    loss.backward()
    torch.cuda.synchronize()
    return [y.detach(), *(s.detach() for s in states), x.grad, *(s.grad for s in hx), *_grads(m.parameters())]


@pytest.mark.parametrize("kind,dtype", [("gru", torch.float32), ("lstm", torch.float32), ("lstmp", torch.float32),
                                        ("tanh", torch.float32), ("relu", torch.float32), ("gru", torch.float16),
                                        ("lstm", torch.bfloat16)])
@pytest.mark.parametrize("train", [False, True])
def test_compile_fullgraph_module_bitwise(kind, dtype, train):
    torch.manual_seed(1)
    m = _seq_module(kind, dtype, dropout=0.3 if train else 0.0).train(train)
    B, T = 5, 9
    HO = 64 if kind == "lstmp" else 128
    x = torch.randn(B, T, 48, device=DEV, dtype=dtype)
    hx = (torch.randn(4, B, HO, device=DEV, dtype=dtype),)
    if kind.startswith("lstm"):
        hx += (torch.randn(4, B, 128, device=DEV, dtype=dtype),)
    compiled = torch.compile(m, fullgraph=True)
    for _ in range(2):   # the second call draws the next dropout mask on both sides
        rng = m._rng_state.clone()
        eager = _run_seq(m, m, x, hx)
        rng_after = m._rng_state.clone()
        m._rng_state.copy_(rng)
        comp = _run_seq(compiled, m, x, hx)
        _assert_same(m._rng_state, rng_after, "rng_state advance")
        for i, (a, b) in enumerate(zip(eager, comp)):
            _assert_same(a, b, f"{kind} {dtype} output/grad #{i}")


@pytest.mark.parametrize("kind", ["gru", "lstm", "tanh", "relu"])
@pytest.mark.parametrize("bias", [True, False])
def test_compile_fullgraph_cell_bitwise(kind, bias):
    import b200rnn

    torch.manual_seed(2)
    cls = {"gru": b200rnn.GRUCell, "lstm": b200rnn.LSTMCell, "tanh": b200rnn.RNNCell, "relu": b200rnn.RNNCell}[kind]
    kw = {"nonlinearity": kind} if kind in ("tanh", "relu") else {}
    cell = cls(40, 48, bias=bias, device=DEV, **kw)
    x0 = torch.randn(6, 40, device=DEV)
    hx0 = (torch.randn(6, 48, device=DEV),) + ((torch.randn(6, 48, device=DEV),) if kind == "lstm" else ())
    compiled = torch.compile(cell, fullgraph=True)

    def run(fn):
        x = x0.clone().requires_grad_(True)
        hx = tuple(s.clone().requires_grad_(True) for s in hx0)
        _zero(cell.parameters())
        out = fn(x, hx if kind == "lstm" else hx[0])
        outs = out if isinstance(out, tuple) else (out,)
        sum((o * (k + 1.5)).sum() for k, o in enumerate(outs)).backward()
        return [*(o.detach() for o in outs), x.grad, *(s.grad for s in hx), *_grads(cell.parameters())]

    for i, (a, b) in enumerate(zip(run(cell), run(compiled))):
        _assert_same(a, b, f"{kind} cell output/grad #{i}")


def test_compile_with_grad_bucket_raises():
    import b200rnn

    m = b200rnn.GRU(64, 128, num_layers=2, device=DEV)
    b200rnn.GradBucket(m)
    with pytest.raises(b200rnn.B200RNNError, match="run it eagerly"):
        torch.compile(m)(torch.randn(5, 3, 64, device=DEV))


# -- the reference's shells -----------------------------------------------------------------------------------------

AUDIO_CFG = dict(num_classes=2, dropout=0.5, rnn_layers=2, embedding_size=256, hidden_dims=256)
TEXT_CFG = dict(num_classes=2, dropout=0.5, rnn_layers=2, embedding_size=1024, hidden_dims=128, bidirectional=True)


@pytest.fixture
def installed():
    """``install()``, and dynamo's ``allow_rnn``: dynamo refuses any module that is an instance of ``torch.nn.GRU`` /
    ``LSTM`` / ``RNN`` as looked up at trace time, which after ``install()`` are the b200rnn classes"""
    import b200rnn

    b200rnn.install()
    with torch._dynamo.config.patch(allow_rnn=True):
        yield b200rnn
    b200rnn.uninstall()


def _ref_model(which):
    from oracle.ref_models import RefAudio, RefText

    torch.manual_seed(3)
    if which == "audio":
        return RefAudio(AUDIO_CFG).to(DEV), torch.randn(4, 12, 256, device=DEV)
    return RefText(TEXT_CFG).to(DEV), torch.randn(4, 7, 1024, device=DEV)


def _rnn_of(model):
    return model.lstm_net_audio if hasattr(model, "lstm_net_audio") else model.lstm_net


def _shell_step(fn, model, x, seed):
    torch.manual_seed(seed)   # the shell's nn.Dropout draws from torch's generator on both sides
    _zero(model.parameters())
    xg = x.clone().requires_grad_(True)
    out = fn(xg)
    (out * torch.tensor([1.0, -2.0], device=DEV)).sum().backward()
    torch.cuda.synchronize()
    return [out.detach(), xg.grad, *_grads(model.parameters())]


@pytest.mark.parametrize("which", ["audio", "text"])
@pytest.mark.parametrize("train", [False, True])
def test_compile_reference_shells_bitwise(installed, which, train):
    import b200rnn

    model, x = _ref_model(which)
    assert isinstance(_rnn_of(model), (b200rnn.GRU, b200rnn.LSTM))
    model.train(train)
    compiled = torch.compile(model, fullgraph=True, backend="aot_eager")
    rng = _rnn_of(model)._rng_state
    for step in range(2):
        before = rng.clone()
        eager = _shell_step(model, model, x, seed=10 + step)
        after = rng.clone()
        rng.copy_(before)
        comp = _shell_step(compiled, model, x, seed=10 + step)
        _assert_same(rng, after, "rng_state advance")
        if train:
            assert not torch.equal(before, after)
        for i, (a, b) in enumerate(zip(eager, comp)):
            _assert_same(a, b, f"{which} train={train} step {step} output/grad #{i}")


# -- b200rnn.models -------------------------------------------------------------------------------------------------

def _close(a, b, rel, what):
    assert (a - b).abs().max().item() <= rel * max(b.abs().max().item(), 1e-30) + 1e-9, what


@pytest.mark.parametrize("which", ["audio", "text"])
def test_compile_models_fullgraph_within_parity(which):
    import b200rnn

    torch.manual_seed(4)
    if which == "audio":
        model, x = b200rnn.AudioBiLSTM(AUDIO_CFG).to(DEV).eval(), torch.randn(4, 12, 256, device=DEV)
    else:
        model, x = b200rnn.TextBiLSTM(TEXT_CFG).to(DEV).eval(), torch.randn(4, 7, 1024, device=DEV)
    compiled = torch.compile(model, fullgraph=True)
    eager = _shell_step(model, model, x, seed=0)
    comp = _shell_step(compiled, model, x, seed=0)
    assert (eager[0] - comp[0]).abs().max().item() < 1e-4
    for i, (a, b) in enumerate(zip(eager[1:], comp[1:])):
        if a is not None:
            _close(b, a, 1e-4, f"{which} grad #{i}")
    explained = torch._dynamo.explain(model)(x)
    assert explained.graph_break_count == 0, explained.break_reasons


class _Features(torch.nn.Module):
    """``pretrained_feature`` of a fusion model on two tensors (the exported entry point)"""

    def __init__(self, net, ref: bool):
        super().__init__()
        self.net, self.ref = net, ref

    def forward(self, audio, text):
        from b200rnn.staging import FuseBatch

        if self.ref:
            return self.net.pretrained_feature_tensors(audio, text)
        return self.net.pretrained_feature(FuseBatch(audio=audio, text=text))


def _fusion_features(ref=False):
    import b200rnn
    from oracle.ref_models import RefFusion

    torch.manual_seed(5)
    net = (RefFusion if ref else b200rnn.fusion_net)(1024, 128, 2, 0.3, 2, 256, 256).to(DEV).eval()
    return _Features(net, ref).eval(), (torch.randn(4, 12, 256, device=DEV), torch.randn(4, 7, 1024, device=DEV))


def test_compile_fusion_features_within_parity():
    feats, args = _fusion_features()
    eager = feats(*args)
    comp = torch.compile(feats, fullgraph=True)(*args)
    for a, b in zip(eager, comp):
        assert (a - b).abs().max().item() < 1e-4
    explained = torch._dynamo.explain(feats)(*args)
    assert explained.graph_break_count == 0, explained.break_reasons


# -- export ---------------------------------------------------------------------------------------------------------

def _export_roundtrip(tmp_path, module, args, name, bitwise=True):
    with torch.no_grad():
        eager = module(*args)
        ep = torch.export.export(module, args)
        assert "b200rnn.rnn_forward" in str(ep.graph)
        out = ep.module()(*args)
    eager = eager if isinstance(eager, tuple) else (eager,)
    out = out if isinstance(out, tuple) else (out,)
    for a, b in zip(eager, out):
        if bitwise:
            _assert_same(a, b, f"{name} exported output")
        else:   # eager takes the shell fusions, the program their unfused expressions
            assert (a - b).abs().max().item() < 1e-4, name
    path = str(tmp_path / f"{name}.pt2")
    torch.export.save(ep, path)
    inputs = str(tmp_path / f"{name}_inputs.pt")
    # the reloaded program must reproduce this one bitwise
    torch.save({"args": [a.cpu() for a in args], "out": [o.cpu() for o in out]}, inputs)
    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "icassp2022-depression_b200")
    script = textwrap.dedent(f"""
        import sys, torch
        sys.path.insert(0, {pkg!r})
        import b200rnn
        ep = torch.export.load({path!r})
        d = torch.load({inputs!r})
        with torch.no_grad():
            out = ep.module()(*[a.cuda() for a in d["args"]])
        out = out if isinstance(out, tuple) else (out,)
        assert all(torch.equal(o.cpu(), r) for o, r in zip(out, d["out"])), "reloaded program differs"
        print("reload ok")
    """)
    proc = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0 and "reload ok" in proc.stdout, proc.stdout + proc.stderr


@pytest.mark.parametrize("which", ["audio", "text"])
def test_export_reference_shells(installed, tmp_path, which):
    model, x = _ref_model(which)
    _export_roundtrip(tmp_path, model.eval(), (x,), which)


def test_export_reference_fusion_features(installed, tmp_path):
    feats, args = _fusion_features(ref=True)
    _export_roundtrip(tmp_path, feats, args, "ref_fusion")


def test_export_fusion_net_features(tmp_path):
    feats, args = _fusion_features()
    _export_roundtrip(tmp_path, feats, args, "fusion", bitwise=False)


# -- CUDA-graph trees -----------------------------------------------------------------------------------------------

def test_reduce_overhead_replays_draw_new_masks():
    import b200rnn

    torch.manual_seed(6)
    m = b200rnn.GRU(64, 128, num_layers=3, dropout=0.5, batch_first=True, device=DEV).train()
    x0 = torch.randn(4, 10, 64, device=DEV)

    def step(x):
        return m(x)

    def loss_of(y, h_n):   # outside the compiled step: inductor's reductions round differently from eager's
        return (y * torch.linspace(-1, 1, y.shape[-1], device=DEV)).sum() + h_n.sum()

    compiled = torch.compile(step, mode="reduce-overhead", fullgraph=True)
    outs = []
    for i in range(4):
        before = m._rng_state.clone()
        _zero(m.parameters())
        x = x0.clone().requires_grad_(True)
        y, h_n = compiled(x)
        comp = [y.detach().clone(), h_n.detach().clone()]
        loss_of(y, h_n).backward()
        comp += [x.grad.clone(), *_grads(m.parameters())]
        after = m._rng_state.clone()
        m._rng_state.copy_(before)
        _zero(m.parameters())
        xe = x0.clone().requires_grad_(True)
        ye, he = step(xe)
        eager = [ye.detach(), he.detach()]
        loss_of(ye, he).backward()
        eager += [xe.grad, *_grads(m.parameters())]
        _assert_same(m._rng_state, after, f"replay {i} rng_state")
        for k, (a, b) in enumerate(zip(eager, comp)):
            _assert_same(a, b, f"replay {i} output/grad #{k}")
        outs.append(comp[0])
    assert not any(torch.equal(outs[i], outs[j]) for i in range(len(outs)) for j in range(i)), \
        "successive replays drew the same dropout masks"
