"""fp32 GRU / LSTM / RNN modules under ``torch.autocast("cuda")``: the 16-bit kernels on the fp32 parameters as masters
(``B200RNN_FLAG_F32_PARAMS``).

The contract: under autocast an fp32 module ``m`` returns exactly what its 16-bit twin ``copy.deepcopy(m).to(dt)``
returns on the input cast to ``dt``, where ``dt`` is the dtype stock torch's RNNs give under the same region; each fp32
``.grad`` is the twin's gradient widened to fp32 (added in fp32 to an existing one), and the input and state gradients
reach the caller's tensors in their dtypes."""
import copy

import pytest
import torch
import torch.nn as nn

import b200rnn
from b200rnn import _lib
from b200rnn.modules import _TORCH_GRU, _TORCH_LSTM, _TORCH_RNN

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
AMP = (torch.float16, torch.bfloat16)
DT = torch.float16   # what stock's autocast wrapper casts to whatever the region's dtype (pinned below)
OURS = {"gru": b200rnn.GRU, "lstm": b200rnn.LSTM, "tanh": b200rnn.RNN, "relu": b200rnn.RNN}
STOCK = {"gru": _TORCH_GRU, "lstm": _TORCH_LSTM, "tanh": _TORCH_RNN, "relu": _TORCH_RNN}


def _kw(kind, I, H=None, **kw):
    if H is not None:
        kw["hidden_size"] = H
    if kind in ("tanh", "relu"):
        kw["nonlinearity"] = kind
    return dict(input_size=I, **kw)


def _pair(kind, seed=0, **kw):
    torch.manual_seed(seed)
    m = OURS[kind](**kw).to(DEV)
    return m, copy.deepcopy(m).to(DT)


def _states(kind, m, B, dtype, seed):
    if B is None:
        return None
    g = torch.Generator(device=DEV).manual_seed(seed)
    L, H = m.num_layers * (2 if m.bidirectional else 1), m.hidden_size
    shape = (L, B, H) if B > 0 else (L, H)
    h = torch.randn(shape, generator=g, device=DEV).to(dtype)
    return (h, torch.randn(shape, generator=g, device=DEV).to(dtype)) if kind == "lstm" else h


def _flat_states(hx):
    return [] if hx is None else (list(hx) if isinstance(hx, tuple) else [hx])


def _outputs(kind, out):
    y, hn = out
    y = y.data if isinstance(y, nn.utils.rnn.PackedSequence) else y
    return [y, *(_flat_states(hn))]


def _run(module, x, hx, amp, weights, packed_lengths=None):
    """forward (under autocast when amp is a dtype) and a backward of sum(out * weight) for every output"""
    xin = x
    if packed_lengths is not None:
        xin = nn.utils.rnn.pack_padded_sequence(x, packed_lengths, batch_first=module.batch_first,
                                                enforce_sorted=False)
    with torch.autocast("cuda", dtype=amp or torch.float16, enabled=amp is not None):
        out = module(xin, hx) if hx is not None else module(xin)
    outs = _outputs(None, out)
    loss = sum((o.float() * w[: o.numel()].view_as(o)).sum() for o, w in zip(outs, weights))
    loss.backward()
    torch.cuda.synchronize()
    return [o.detach() for o in outs]


def _weights_for(outs_shapes, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(n, generator=g, device=DEV).to(DT).float() for n in outs_shapes]


def _check_twin(kind, amp, T=7, B=5, I=48, seed=0, hx_dtype=None, unbatched=False, packed=False, accumulate=False,
                train=True, **kw):
    m, twin = _pair(kind, seed, **_kw(kind, I, **kw))
    m.train(train)
    twin.train(train)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    bf = m.batch_first
    shape = (T, I) if unbatched else ((B, T, I) if bf else (T, B, I))
    x = torch.randn(shape, generator=g, device=DEV)
    x32 = x.clone().requires_grad_(True)
    x16 = x.to(DT).requires_grad_(True)
    hx32 = hx16 = None
    if hx_dtype is not None:
        hb = 0 if unbatched else B
        base = _states(kind, m, hb, torch.float32, seed + 2)
        leaf = lambda s, dt: s.to(dt).clone().requires_grad_(True)  # noqa: E731
        hx32 = tuple(leaf(s, hx_dtype) for s in base) if kind == "lstm" else leaf(base, hx_dtype)
        hx16 = tuple(leaf(s, DT) for s in base) if kind == "lstm" else leaf(base, DT)
    lengths = None
    if packed:
        lengths = torch.tensor([T, 3, T - 1, 1, 4][:B])
    old = None
    if accumulate:
        old = [torch.randn_like(p) for p in m.parameters()]
        for p, o in zip(m.parameters(), old):
            p.grad = o.clone()
    with torch.no_grad():
        shapes = [o.numel() for o in _outputs(kind, twin(x16 if lengths is None else
                                                          nn.utils.rnn.pack_padded_sequence(
                                                              x16, lengths, batch_first=bf, enforce_sorted=False),
                                                          hx16))]
    # the probe above advanced the twin's Philox offset; restart both from the same state
    twin._rng_state.copy_(m._rng_state)
    w = _weights_for(shapes, seed + 3)
    ours = _run(m, x32, hx32, amp, w, lengths)
    ref = _run(twin, x16, hx16, None, w, lengths)
    for a, b in zip(ours, ref):
        assert a.dtype == DT and torch.equal(a, b)
    for i, (p, q) in enumerate(zip(m.parameters(), twin.parameters())):
        assert p.grad.dtype == torch.float32
        want = q.grad.float() if old is None else old[i] + q.grad.float()
        assert torch.equal(p.grad, want), i
    assert x32.grad.dtype == torch.float32 and torch.equal(x32.grad, x16.grad.float())
    for s32, s16 in zip(_flat_states(hx32), _flat_states(hx16)):
        assert s32.grad.dtype == s32.dtype and torch.equal(s32.grad, s16.grad.to(s32.dtype))
    assert torch.equal(m._rng_state, twin._rng_state)


CASES = [
    ("gru", dict(hidden_size=256)),                          # fixed config
    ("gru", dict(hidden_size=96)),
    ("lstm", dict(hidden_size=128)),                         # fixed config
    ("lstm", dict(hidden_size=320)),
    ("tanh", dict(hidden_size=64)),
    ("relu", dict(hidden_size=64)),
    ("gru", dict(hidden_size=768)),                          # runtime-sized, 16-bit L2 tier
    ("gru", dict(hidden_size=256, num_layers=2, bidirectional=True, dropout=0.3, batch_first=True)),
    ("lstm", dict(hidden_size=128, num_layers=2, bidirectional=True, dropout=0.3)),
    ("relu", dict(hidden_size=64, num_layers=2, bidirectional=True, dropout=0.3, batch_first=True)),
    ("lstm", dict(hidden_size=320, num_layers=2, dropout=0.3, batch_first=True)),
]


@pytest.mark.parametrize("amp", AMP)
@pytest.mark.parametrize("kind,kw", CASES)
def test_twin_equality_bitwise(kind, kw, amp):
    _check_twin(kind, amp, **kw)


@pytest.mark.parametrize("amp", AMP)
@pytest.mark.parametrize("kind,kw", [CASES[0], CASES[2], CASES[3], CASES[5], CASES[8]])
def test_twin_equality_accumulated_eval_packed_and_states(kind, kw, amp):
    _check_twin(kind, amp, accumulate=True, **kw)
    _check_twin(kind, amp, train=False, **kw)
    _check_twin(kind, amp, packed=True, **kw)
    _check_twin(kind, amp, hx_dtype=torch.float32, **kw)
    _check_twin(kind, amp, hx_dtype=DT, **kw)
    _check_twin(kind, amp, unbatched=True, hx_dtype=torch.float32, **kw)


def test_config_under_autocast_and_nested_disabled_region():
    m = b200rnn.LSTM(16, 32, num_layers=2).to(DEV)
    x = torch.randn(3, 2, 16, device=DEV)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert m._autocast_dtype() == DT and m._config(DT).master_f32
        assert b200rnn.GRU(16, 32).to(DEV).half()._autocast_dtype() is None
        with torch.autocast("cuda", enabled=False):
            assert m._autocast_dtype() is None
            y_off = m(x)[0]
    assert y_off.dtype == torch.float32 and torch.equal(y_off, m(x)[0])   # exactly the fp32 path
    # a 16-bit module keeps its dtype under autocast
    h = b200rnn.GRU(16, 32).to(DEV).to(torch.bfloat16)
    with torch.autocast("cuda", dtype=torch.float16):
        assert h(x.to(torch.bfloat16))[0].dtype == torch.bfloat16


# -- parity with stock torch under the same region ------------------------------------------------------------------

@pytest.mark.parametrize("amp", AMP)
@pytest.mark.parametrize("kind", ["gru", "lstm", "tanh"])
def test_output_dtypes_and_mixed_inputs_match_stock(kind, amp):
    torch.manual_seed(0)
    stock = STOCK[kind](**_kw(kind, 16, 32, num_layers=2)).to(DEV)
    ours = b200rnn.from_torch(stock).to(DEV)
    x = torch.randn(4, 3, 16, device=DEV)
    for xd in (torch.float32, torch.float16, torch.bfloat16):
        for hd in (None, torch.float32, torch.float16):
            hx = None if hd is None else _states(kind, ours, 3, hd, 1)
            with torch.autocast("cuda", dtype=amp):
                so = _raised(lambda: stock(x.to(xd), hx)) or _outputs(kind, stock(x.to(xd), hx))
                oo = _raised(lambda: ours(x.to(xd), hx)) or _outputs(kind, ours(x.to(xd), hx))
            if isinstance(so, tuple):   # stock refuses the combination: so do we, with its exception type
                assert isinstance(oo, tuple) and oo[0] is so[0], (xd, hd, so, oo)
                continue
            assert [t.dtype for t in oo] == [t.dtype for t in so], (xd, hd)
            assert so[0].dtype == DT   # the dtype stock's autocast wrapper runs in: float16 in either region


def _raised(fn):
    try:
        fn()
    except Exception as e:   # noqa: BLE001 - the type and message are what is compared
        return type(e), str(e)
    return None


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_errors_under_autocast_match_stock(kind):
    torch.manual_seed(0)
    stock = STOCK[kind](**_kw(kind, 16, 32)).to(DEV)
    ours = b200rnn.from_torch(stock).to(DEV)
    bad = [
        lambda m: m(torch.randn(4, 3, 15, device=DEV)),                            # input_size
        lambda m: m(torch.randn(4, 3, 16, 1, device=DEV)),                          # rank
        lambda m: m(torch.randn(4, 3, 16, device=DEV), _states(kind, ours, 2, torch.float32, 0)),   # hx batch
        lambda m: m(torch.randn(4, 3, 16, device=DEV), _states(kind, ours, 0, torch.float32, 0)),   # hx rank
    ]
    for f in bad:
        with torch.autocast("cuda", dtype=torch.float16):
            s, o = _raised(lambda: f(stock)), _raised(lambda: f(ours))
        assert s is not None and o is not None
        assert o[0] is s[0] and o[1].replace(type(ours).__name__, type(stock).__name__) == s[1], (o, s)


# -- GradScaler ------------------------------------------------------------------------------------------------------

def _amp_model(rnn_cls):
    torch.manual_seed(5)
    return nn.ModuleDict({"fc": nn.Linear(24, 32), "rnn": rnn_cls(32, 128, num_layers=2),
                          "out": nn.Linear(128, 1)}).to(DEV)


def _amp_steps(model, n, scale):
    opt = torch.optim.SGD(model.parameters(), lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=scale, growth_interval=1000)
    g = torch.Generator(device=DEV).manual_seed(9)
    x = torch.randn(10, 8, 24, generator=g, device=DEV)
    log = []
    for _ in range(n):
        before = [p.detach().clone() for p in model["rnn"].parameters()]
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            h = model["fc"](x)
            y = model["rnn"](h)[0]
            loss = model["out"](y).float().square().mean()
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        moved = any(not torch.equal(a, p) for a, p in zip(before, model["rnn"].parameters()))
        log.append((scaler.get_scale(), moved))
    return log


def test_grad_scaler_skips_overflowed_steps_like_stock():
    ours = _amp_steps(_amp_model(b200rnn.LSTM), 30, 2.0 ** 30)
    stock = _amp_steps(_amp_model(_TORCH_LSTM), 30, 2.0 ** 30)
    # 2^30 overflows the fp16 gradients: the step is skipped and the scale halves, as with stock
    assert ours[0] == (2.0 ** 29, False) and stock[0] == (2.0 ** 29, False)
    assert [s for s, _ in ours[:2]] == [s for s, _ in stock[:2]]
    # once the scale is small enough the steps are taken and move the parameters
    assert ours[-1][1] and stock[-1][1]
    assert any(mv for _, mv in ours)


# -- launches and casts ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,kw", [CASES[0], CASES[3], CASES[8]])
def test_launch_counts_and_no_per_weight_casts(kind, kw):
    m, twin = _pair(kind, **_kw(kind, 48, **kw))
    x = torch.randn(6, 5, 48, device=DEV)
    if m.batch_first:
        x = x.transpose(0, 1).contiguous()
    with torch.autocast("cuda", dtype=torch.float16):
        m(x)  # warm-up
    twin(x.to(DT))
    counts = {}
    for name, mod, amp in (("ours", m, True), ("twin", twin, False)):
        xi = (x if amp else x.to(DT)).requires_grad_(True)
        torch.cuda.synchronize()
        c0 = _lib.launch_count()
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            y = mod(xi)[0]
        c1 = _lib.launch_count()
        y.float().sum().backward()
        torch.cuda.synchronize()
        counts[name] = (c1 - c0, _lib.launch_count() - c1)
    assert counts["ours"][0] <= counts["twin"][0] + 1, counts
    assert counts["ours"][1] < counts["twin"][1], counts
    from torch.profiler import ProfilerActivity, profile
    copies = []
    for mod, amp in ((m, True), (twin, False)):
        with profile(activities=[ProfilerActivity.CPU]) as prof:
            xi = x.clone().requires_grad_(True)
            with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                y = mod(xi if amp else xi.to(DT))[0]
            y.float().sum().backward()
            torch.cuda.synchronize()
        copies.append(sum(e.count for e in prof.key_averages() if e.key == "aten::_to_copy"))
    # the casts of the input, of its gradient and of the loss, as around the twin: none per weight
    assert copies[0] == copies[1], copies


# -- CUDA graphs, torch.compile, torch.export ------------------------------------------------------------------------

def _step(m, x):
    with torch.autocast("cuda", dtype=torch.float16):
        y, *_ = m(x)
    loss = (y.float() * torch.linspace(-1, 1, y.size(-1), device=DEV)).sum()
    # y detached: a live autograd graph would keep its AccumulateGrad nodes on the stream they were made on
    return [y.detach(), *torch.autograd.grad(loss, [x, *m.parameters()])]


@pytest.mark.parametrize("kind,kw", [CASES[0], CASES[3], CASES[9]])
def test_cuda_graph_capture_replays_eager(kind, kw):
    m, _ = _pair(kind, **_kw(kind, 48, **{**kw, "dropout": 0.0}))
    x = torch.randn(6, 5, 48, device=DEV)
    if m.batch_first:
        x = x.transpose(0, 1).contiguous()
    xs = x.clone().requires_grad_(True)
    eager = _step(m, xs)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _step(m, xs)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static = _step(m, xs)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


@pytest.mark.parametrize("kind,kw", [CASES[0], CASES[8]])
def test_compile_and_export_under_autocast_equal_eager(kind, kw):
    m, _ = _pair(kind, **_kw(kind, 48, **{**kw, "dropout": 0.0}))
    m.eval()
    x = torch.randn(6, 5, 48, device=DEV)
    if m.batch_first:
        x = x.transpose(0, 1).contiguous()
    xs = x.clone().requires_grad_(True)
    eager = _step(m, xs)
    torch._dynamo.reset()
    with torch._dynamo.config.patch(allow_rnn=True):
        cm = torch.compile(m, fullgraph=True)
        compiled = _step(cm, xs)
    for a, b in zip(compiled, eager):
        assert a.dtype == b.dtype and torch.equal(a, b)
    with torch.no_grad():
        with torch.autocast("cuda", dtype=torch.float16):
            ep = torch.export.export(m, (x,))
            exported = ep.module()(x)[0]
            want = m(x)[0]
    assert exported.dtype == DT and torch.equal(exported, want)


# -- model shells ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("grad", [False, True])
def test_forward_ln_sum_under_autocast_is_the_unfused_expression(grad):
    torch.manual_seed(2)
    m = b200rnn.GRU(256, 256, num_layers=2, batch_first=True).to(DEV).eval()
    ln = nn.LayerNorm(256).to(DEV)
    x = torch.randn(4, 9, 256, device=DEV)
    outs = []
    for fused in (True, False):
        m.zero_grad()
        xs = x.clone().requires_grad_(grad)
        with torch.set_grad_enabled(grad), torch.autocast("cuda", dtype=torch.float16):
            out = m.forward_ln_sum(xs, ln) if fused else m(ln(xs))[0].sum(dim=1)
        r = [out.detach()]
        if grad:
            out.float().sum().backward()
            r += [xs.grad, *(p.grad for p in m.parameters())]
        outs.append(r)
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("which", ["audio", "text"])
def test_reference_classes_under_autocast_match_stock_dtypes(which):
    from oracle.ref_models import RefAudio, RefText

    cfgs = {"audio": (RefAudio, dict(num_classes=2, dropout=0.5, rnn_layers=2, embedding_size=256, hidden_dims=256),
                      (4, 12, 256)),
            "text": (RefText, dict(num_classes=2, dropout=0.5, rnn_layers=2, embedding_size=1024, hidden_dims=128,
                                   bidirectional=True), (4, 7, 1024))}
    cls, cfg, shape = cfgs[which]
    x = torch.randn(shape, device=DEV)
    dtypes = []
    for install in (False, True):
        if install:
            b200rnn.install()
        try:
            torch.manual_seed(3)
            model = cls(cfg).to(DEV)
            xs = x.clone().requires_grad_(True)
            with torch.autocast("cuda", dtype=torch.float16):
                out = model(xs)
            out.float().sum().backward()
            torch.cuda.synchronize()
            rnn = model.lstm_net_audio if which == "audio" else model.lstm_net
            assert isinstance(rnn, (b200rnn.GRU, b200rnn.LSTM)) == install
            assert all(p.grad is not None and p.grad.dtype == torch.float32 for p in rnn.parameters())
            dtypes.append((out.dtype, xs.grad.dtype))
        finally:
            b200rnn.uninstall()
    assert dtypes[0] == dtypes[1]
