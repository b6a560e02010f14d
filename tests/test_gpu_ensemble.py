"""Ensembles and per-sample gradients under torch.func on the GPU (b200rnn/func.py, RecModels in csrc/rnn_anyh.cu).

Every vmapped call is checked against a Python loop of single-model eager calls with the same inputs and loss weights:
outputs, h_n / c_n and every gradient (weights, x, hx). Where a single model already runs the runtime-sized kernels
(hidden sizes other than 128 / 256, and the Elman modes everywhere) the ensemble must be bitwise equal to the loop. At
128 / 256 the loop runs the fixed configs and the ensemble the runtime-sized kernels; both are held to float64 (stock
torch on CPU) by the other suites, with outputs within 1e-5 and gradients within 1e-4 of the largest entry
(tests/test_gpu_any_hidden.py), so here they must agree within twice those bounds."""
import copy

import pytest
import torch
from torch.func import functional_call, grad, stack_module_state, vmap

import b200rnn
from b200rnn import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KINDS = ("gru", "lstm", "rnn_tanh", "rnn_relu")


def _ctor(kind):
    if kind.startswith("rnn_"):
        return lambda *a, **k: b200rnn.RNN(*a, nonlinearity=kind[4:], **k)
    return b200rnn.GRU if kind == "gru" else b200rnn.LSTM


def _bitwise(kind, H):
    return kind.startswith("rnn_") or H not in (128, 256)


def _models(kind, M, I, H, L=1, bi=False, bf=False, dropout=0.0, seed=0):
    torch.manual_seed(seed)
    return [_ctor(kind)(I, H, num_layers=L, bidirectional=bi, batch_first=bf, dropout=dropout).to(DEV)
            for _ in range(M)]


def _states(kind, n, L, D, B, H, seed=3):
    g = torch.Generator().manual_seed(seed)
    mk = lambda: (0.5 * torch.randn(*n, L * D, B, H, generator=g)).to(DEV)  # noqa: E731
    return (mk(), mk()) if kind == "lstm" else mk()


def _loss(out, ws):
    return sum((o * w).sum() for o, w in zip(out, ws))


def _check(kind, H, a, b, what, grad=False):
    if _bitwise(kind, H):
        assert torch.equal(a, b), (what, (a - b).abs().max().item())
    elif grad:
        err = ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()
        assert err <= 2e-4, (what, err)
    else:
        assert (a - b).abs().max().item() <= 2e-5, what


def _run_ensemble(models, x, hx, x_batched, hx_mode, randomness="error"):
    """vmap over the stacked models; returns (outputs, stacked params, x, hx) with gradients taken outside vmap"""
    params, bufs = stack_module_state(models)
    base = copy.deepcopy(models[0])

    def f(p, b, xx, hh):
        return functional_call(base, (p, b), (xx, hh))

    hx_dim = None if hx is None or hx_mode == "shared" else 0
    out = vmap(f, in_dims=(0, 0, 0 if x_batched else None, hx_dim), randomness=randomness)(params, bufs, x, hx)
    return out, params, bufs


def _flat_out(out):
    y, st = out
    return [y, *(st if isinstance(st, tuple) else (st,))]


def _compare_with_loop(kind, M, I, H, L, bi, bf, B=5, T=6, hx_mode="none", x_batched=True, seed=0):
    D = 2 if bi else 1
    models = _models(kind, M, I, H, L, bi, bf, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    xs = (torch.randn(M, B, T, I, generator=g) if bf else torch.randn(M, T, B, I, generator=g)).to(DEV)
    x = (xs if x_batched else xs[0]).clone().requires_grad_(True)
    hx = None
    if hx_mode != "none":
        hx = _states(kind, (M,) if hx_mode == "batched" else (), L, D, B, H)
        hx = tuple(s.requires_grad_(True) for s in hx) if kind == "lstm" else hx.requires_grad_(True)
    out, params, _ = _run_ensemble(models, x, hx, x_batched, hx_mode)
    flat = _flat_out(out)
    ws = [torch.randn(o.shape, generator=g).to(DEV) for o in flat]
    _loss(flat, ws).backward()
    hx_list = [] if hx is None else (list(hx) if kind == "lstm" else [hx])

    dx_loop = torch.zeros_like(x)
    dh_loop = [torch.zeros_like(s) for s in hx_list]
    for m, model in enumerate(models):
        xm = (x[m] if x_batched else x).detach().clone().requires_grad_(True)
        hm = None
        if hx is not None:
            pick = (lambda s: s[m]) if hx_mode == "batched" else (lambda s: s)
            hs = [pick(s).detach().clone().requires_grad_(True) for s in hx_list]
            hm = tuple(hs) if kind == "lstm" else hs[0]
        ref = _flat_out(model(xm, hm))
        for o, r, name in zip(flat, ref, ("y", "h_n", "c_n")):
            _check(kind, H, o[m].detach(), r.detach(), f"model {m} {name}")
        _loss(ref, [w[m] for w in ws]).backward()
        for n, p in model.named_parameters():
            _check(kind, H, params[n].grad[m], p.grad, f"model {m} d{n}", grad=True)
        if x_batched:
            _check(kind, H, x.grad[m], xm.grad, f"model {m} dx", grad=True)
        else:
            dx_loop += xm.grad
        if hx is not None:
            for i, s in enumerate(hs):
                if hx_mode == "batched":
                    _check(kind, H, hx_list[i].grad[m], s.grad, f"model {m} dh_0[{i}]", grad=True)
                else:
                    dh_loop[i] += s.grad
    # a shared x / hx gathers every model's gradient (summed over the models in order, as the loop sums here)
    if not x_batched:
        torch.testing.assert_close(x.grad, dx_loop, rtol=1e-5, atol=1e-6)
    if hx_mode == "shared":
        for s, r in zip(hx_list, dh_loop):
            torch.testing.assert_close(s.grad, r, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("H", (64, 128, 208, 256))
@pytest.mark.parametrize("L,bi,bf", ((1, False, False), (2, True, True), (3, False, True)))
def test_ensemble_matches_loop(kind, H, L, bi, bf):
    _compare_with_loop(kind, 3, 24, H, L, bi, bf)


@pytest.mark.parametrize("kind", ("gru", "lstm", "rnn_tanh"))
@pytest.mark.parametrize("hx_mode", ("none", "batched", "shared"))
@pytest.mark.parametrize("x_batched", (True, False))
def test_ensemble_hx_and_shared_x(kind, hx_mode, x_batched):
    _compare_with_loop(kind, 3, 16, 64, 2, True, False, hx_mode=hx_mode, x_batched=x_batched)


@pytest.mark.parametrize("kind,M,H", (("gru", 1, 64), ("lstm", 8, 64), ("rnn_relu", 8, 208), ("lstm", 3, 512),
                                      ("gru", 8, 256)))
def test_ensemble_model_counts_and_wide_hidden(kind, M, H):
    _compare_with_loop(kind, M, 32, H, 2, True, True, B=8, T=3)


def test_ensemble_in_several_waves_matches_loop():
    """12 bidirectional GRU-64 models at B = 64: 12 x 2 x 16 clusters of 2 CTAs, more than one wave holds on a 132-SM
    card, so the later models' clusters wait for earlier ones to finish"""
    _compare_with_loop("gru", 12, 16, 64, 1, True, False, B=64, T=3)


@pytest.mark.parametrize("kind", ("gru", "lstm"))
@pytest.mark.parametrize("H", (128, 256))
def test_ensemble_at_fixed_config_sizes_vs_float64(kind, H):
    """At 128 / 256 each model of the ensemble against stock torch in float64 on the CPU, with the bounds the
    runtime-sized kernels meet at every other size (tests/test_gpu_any_hidden.py): outputs within 1e-5, gradients within
    1e-4 of the largest entry"""
    M, B, T, I, L = 3, 5, 6, 24, 2
    models = _models(kind, M, I, H, L, True)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(M, T, B, I, generator=g).to(DEV).requires_grad_(True)
    out, params, _ = _run_ensemble(models, x, None, True, "none")
    flat = _flat_out(out)
    ws = [torch.randn(o.shape, generator=g).to(DEV) for o in flat]
    _loss(flat, ws).backward()
    stock = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    rel = lambda a, b: ((a.detach().double().cpu() - b).abs().max() / b.abs().max()).item()  # noqa: E731
    for m, model in enumerate(models):
        ref = stock(I, H, num_layers=L, bidirectional=True).double()
        ref.load_state_dict({k: v.detach().double().cpu() for k, v in model.state_dict().items()})
        xr = x[m].detach().double().cpu().requires_grad_(True)
        r = _flat_out(ref(xr))
        for o, rr in zip(flat, r):
            assert (o[m].detach().double().cpu() - rr.detach()).abs().max().item() <= 1e-5, m
        _loss(r, [w[m].double().cpu() for w in ws]).backward()
        assert rel(x.grad[m], xr.grad) <= 1e-4, m
        for n, p in ref.named_parameters():
            assert rel(params[n].grad[m], p.grad) <= 1e-4, (m, n)


@pytest.mark.parametrize("kind", ("gru", "lstm"))
def test_perturbing_one_model_changes_only_its_outputs_and_gradients(kind):
    M, B, T, I, H = 4, 3, 5, 16, 64
    models = _models(kind, M, I, H, 2, True)
    x = torch.randn(M, T, B, I, device=DEV)

    def run(ms):
        params, bufs = stack_module_state(ms)
        base = copy.deepcopy(ms[0])
        out = vmap(lambda p, b, xx: functional_call(base, (p, b), (xx,)))(params, bufs, x)
        out[0].square().sum().backward()
        return out[0].detach(), {n: p.grad for n, p in params.items()}

    y0, g0 = run(models)
    with torch.no_grad():
        models[2].weight_hh_l1.add_(0.05)
    y1, g1 = run(models)
    for m in range(M):
        same = m != 2
        assert torch.equal(y0[m], y1[m]) == same, m
        assert all(torch.equal(g0[n][m], g1[n][m]) for n in g0) == same, m


def test_plain_grad_equals_eager_backward():
    for kind in KINDS:
        model = _models(kind, 1, 16, 96, 2, True)[0]
        x = torch.randn(7, 4, 16, device=DEV)
        params = {n: p.detach() for n, p in model.named_parameters()}
        bufs = dict(model.named_buffers())

        def loss(p, xx):
            y, _ = functional_call(model, (p, bufs), (xx,))
            return (y * y.detach().cos()).sum()

        g, dx = grad(loss, argnums=(0, 1))(params, x)
        xe = x.clone().requires_grad_(True)
        y, _ = model(xe)
        (y * y.detach().cos()).sum().backward()
        for n, p in model.named_parameters():
            assert torch.equal(g[n], p.grad), (kind, n)
        assert torch.equal(dx, xe.grad), kind
        v, _ = torch.func.grad_and_value(loss)(params, x)
        assert all(torch.equal(v[n], g[n]) for n in g)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("H", (64, 128))
def test_per_sample_gradients(kind, H):
    N, T, I = 6, 5, 12
    model = _models(kind, 1, I, H, 2, False)[0]
    params = {n: p.detach() for n, p in model.named_parameters()}
    bufs = dict(model.named_buffers())
    xs = torch.randn(N, T, I, device=DEV)
    ts = torch.randn(N, T, H, device=DEV)

    def loss(p, xx, tt):
        y, _ = functional_call(model, (p, bufs), (xx.unsqueeze(1),))
        return ((y.squeeze(1) - tt) ** 2).sum()

    per = vmap(grad(loss), in_dims=(None, 0, 0))(params, xs, ts)
    for n in range(N):
        model.zero_grad()
        y, _ = model(xs[n].unsqueeze(1))
        ((y.squeeze(1) - ts[n]) ** 2).sum().backward()
        for name, p in model.named_parameters():
            _check(kind, H, per[name][n], p.grad, f"sample {n} d{name}", grad=True)


@pytest.mark.parametrize("kind", ("gru", "lstm", "rnn_tanh"))
def test_vmap_of_grad_over_an_ensemble(kind):
    M, B, T, I, H = 3, 4, 5, 16, 80
    models = _models(kind, M, I, H, 2, True)
    params, bufs = stack_module_state(models)
    params = {n: p.detach() for n, p in params.items()}
    base = copy.deepcopy(models[0])
    x = torch.randn(M, T, B, I, device=DEV)

    def loss(p, b, xx):
        y, _ = functional_call(base, (p, b), (xx,))
        return y.sin().sum()

    g = vmap(grad(loss))(params, bufs, x)
    for m, model in enumerate(models):
        y, _ = model(x[m])
        y.sin().sum().backward()
        for n, p in model.named_parameters():
            assert torch.equal(g[n][m], p.grad), (m, n)


def _dropout_models(kind, M):
    return _models(kind, M, 16, 64, 3, True, dropout=0.4, seed=5)


@pytest.mark.parametrize("kind", ("gru", "lstm", "rnn_relu"))
def test_dropout_different_batched_state_matches_loop(kind):
    M = 3
    models = _dropout_models(kind, M)
    for m in models:
        m.train()
    x = torch.randn(M, 6, 4, 16, device=DEV)
    params, bufs = stack_module_state(models)
    base = copy.deepcopy(models[0])
    out = vmap(lambda p, b, xx: functional_call(base, (p, b), (xx,)), randomness="different")(params, bufs, x)
    out[0].sum().backward()
    for m, model in enumerate(models):
        y, _ = model(x[m])
        y.sum().backward()
        assert torch.equal(out[0][m], y), m
        assert torch.equal(bufs["_rng_state"][m], model._rng_state), m
        for n, p in model.named_parameters():
            assert torch.equal(params[n].grad[m], p.grad), (m, n)


def test_dropout_different_shared_state_draws_consecutive_masks():
    M = 3
    models = _dropout_models("gru", M)
    probe = copy.deepcopy(models[0])   # one module: its state serves every model
    state0 = probe._rng_state.clone()
    x = torch.randn(M, 6, 4, 16, device=DEV)
    params, _ = stack_module_state(models)
    bufs = {"_rng_state": probe._rng_state}
    y = vmap(lambda p, xx: functional_call(probe, (p, bufs), (xx,)), in_dims=(0, 0), randomness="different")(params, x)
    end = probe._rng_state.clone()
    probe._rng_state.copy_(state0)
    for m, model in enumerate(models):
        model._rng_state.copy_(probe._rng_state)
        ref, _ = model(x[m])
        probe._rng_state.copy_(model._rng_state)
        assert torch.equal(y[0][m], ref), m
    assert torch.equal(end, probe._rng_state)


def test_dropout_same_applies_one_mask():
    M = 3
    models = _dropout_models("lstm", M)
    probe = copy.deepcopy(models[0])
    state0 = probe._rng_state.clone()
    x = torch.randn(M, 6, 4, 16, device=DEV)
    params, _ = stack_module_state(models)
    bufs = {"_rng_state": probe._rng_state}
    y = vmap(lambda p, xx: functional_call(probe, (p, bufs), (xx,)), randomness="same")(params, x)
    for m, model in enumerate(models):
        model._rng_state.copy_(state0)
        ref, _ = model(x[m])
        assert torch.equal(y[0][m], ref), m
        assert torch.equal(probe._rng_state, model._rng_state), m
    with pytest.raises(_lib.B200RNNError, match="randomness='same'"):
        stacked = stack_module_state(models)
        vmap(lambda p, b, xx: functional_call(probe, (p, b), (xx,)), randomness="same")(*stacked, x)


def test_dropout_error_mode_raises_torchs_message():
    models = _dropout_models("gru", 2)
    params, bufs = stack_module_state(models)
    base = copy.deepcopy(models[0])
    x = torch.randn(2, 6, 4, 16, device=DEV)
    with pytest.raises(RuntimeError, match="vmap: called random operation while in randomness error mode"):
        vmap(lambda p, b, xx: functional_call(base, (p, b), (xx,)))(params, bufs, x)
    base.eval()   # no dropout in eval mode: any randomness works
    vmap(lambda p, b, xx: functional_call(base, (p, b), (xx,)))(params, bufs, x)


def test_out_of_scope_cases_raise():
    x = torch.randn(2, 5, 3, 32, device=DEV)
    cases = [
        (b200rnn.LSTM(32, 128, proj_size=32).to(DEV), x, "proj_size"),
        (b200rnn.GRU(32, 64).to(DEV).half(), x.half(), "float32"),
    ]
    for model, xx, msg in cases:
        params, bufs = stack_module_state([model, copy.deepcopy(model)])
        with pytest.raises(_lib.B200RNNError, match=msg):
            vmap(lambda p, b, xi: functional_call(model, (p, b), (xi,)))(params, bufs, xx)
    model = b200rnn.GRU(32, 64).to(DEV)
    params, bufs = stack_module_state([model, copy.deepcopy(model)])
    with torch.autocast("cuda"), pytest.raises(_lib.B200RNNError, match="autocast"):
        vmap(lambda p, b, xi: functional_call(model, (p, b), (xi,)))(params, bufs, x)
    packed = torch.nn.utils.rnn.pack_padded_sequence(x[0], torch.tensor([5, 4, 2]))
    with pytest.raises(_lib.B200RNNError, match="PackedSequence"):
        grad(lambda p: functional_call(model, (p, bufs), (packed,))[0].data.sum())(dict(model.named_parameters()))


def test_one_recurrence_launch_per_layer_for_the_whole_ensemble():
    M, L = 8, 3
    models = _models("gru", M, 32, 128, L, True)
    params, bufs = stack_module_state(models)
    base = copy.deepcopy(models[0])
    x = torch.randn(M, 3, 8, 32, device=DEV)
    f = vmap(lambda p, b, xx: functional_call(base, (p, b), (xx,)))
    f(params, bufs, x)[0].sum().backward()   # warm
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        f(params, bufs, x)[0].sum().backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert sum("anyh_fwd_kernel" in n for n in names) == L, names
    assert sum("anyh_bwd_kernel" in n for n in names) == L, names
    assert not any("rec_fwd" in n or "rec_bwd" in n for n in names)


def test_cuda_graph_replay_of_a_vmapped_forward_backward():
    M = 3
    models = _models("lstm", M, 16, 64, 2, True)
    params, bufs = stack_module_state(models)
    params = {n: p.detach() for n, p in params.items()}
    base = copy.deepcopy(models[0])
    x = torch.randn(M, 5, 4, 16, device=DEV)

    def step(xx):
        return vmap(grad(lambda p, b, xi: functional_call(base, (p, b), (xi,))[0].tanh().sum()))(params, bufs, xx)

    eager = step(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    static_x = x.clone()
    with torch.cuda.graph(graph):
        out = step(static_x)
    graph.replay()
    torch.cuda.synchronize()
    for n in eager:
        assert torch.equal(out[n], eager[n]), n
