"""Initial state hx: GRU.forward(input, h_0) / LSTM.forward(input, (h_0, c_0)) and the gradients w.r.t. h_0 / c_0.

Oracle: stock torch.nn.GRU / LSTM on CPU with the same hx. Tolerances as tests/test_gpu_varlen.py: outputs and states
1e-5 absolute, gradients 1e-4 relative to the largest entry. The loss covers y, h_n and c_n, so dh_0 / dc_0 see every
path (through the outputs, the final state and the first step's gates). GRU-256 batch sizes reach each forward config
(B = 16: bs2, 64: bs4, 128: tc8 with the streamed projection, 160: tc8 after its GEMM), the wide batches reach the
several-wave fallbacks of tests/test_gpu_coverage.py."""
import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OUT_TOL = 1e-5
GRAD_RTOL = 1e-4
TF32_GRAD_RTOL = 2e-3   # two single-pass TF32 computations of one gradient (test_chunked_equals_whole)


def _models(kind, I, H, L, bi, seed=0):
    import b200rnn

    torch.manual_seed(seed)
    cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    ref = cls(I, H, num_layers=L, bidirectional=bi, batch_first=True)
    return ref, b200rnn.from_torch(ref).to(DEV)


def _states(out):
    return out[1] if isinstance(out[1], tuple) else (out[1],)


def _inputs(kind, B, T, I, H, L, bi, seed=11):
    g = torch.Generator().manual_seed(seed)
    D = 2 if bi else 1
    ns = 1 if kind == "gru" else 2
    x = torch.randn(B, T, I, generator=g)
    hx = [0.5 * torch.randn(L * D, B, H, generator=g) for _ in range(ns)]
    wy = torch.randn(B, T, D * H, generator=g)
    ws = [torch.randn(L * D, B, H, generator=g) for _ in range(ns)]
    return x, hx, wy, ws


def _run(model, x, hx, wy, ws, dev, lens=None, hx_grad=True):
    """padded output, final states, dx, parameter gradients and hx gradients of sum(y * wy) + sum(state * ws)"""
    model.zero_grad(set_to_none=True)
    xx = x.clone().to(dev).requires_grad_(True)
    h0 = [h.clone().to(dev).requires_grad_(hx_grad) for h in hx]
    inp = xx if lens is None else pack_padded_sequence(xx, lens, batch_first=True, enforce_sorted=False)
    out = model(inp, h0[0] if len(h0) == 1 else tuple(h0))
    y = out[0] if lens is None else pad_packed_sequence(out[0], batch_first=True, total_length=x.shape[1])[0]
    loss = (y * wy.to(dev)).sum()
    for s, w in zip(_states(out), ws):
        loss = loss + (s * w.to(dev)).sum()
    loss.backward()
    cpu = lambda t: None if t is None else t.detach().cpu()  # noqa: E731
    return (cpu(y), [cpu(s) for s in _states(out)], cpu(xx.grad), [cpu(p.grad) for p in model.parameters()],
            [cpu(h.grad) for h in h0])


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _compare(mine, ref, names=None):
    y_m, s_m, dx_m, gp_m, gh_m = mine
    y_r, s_r, dx_r, gp_r, gh_r = ref
    assert (y_m - y_r).abs().max().item() <= OUT_TOL
    for a, b in zip(s_m, s_r):
        assert (a - b).abs().max().item() <= OUT_TOL
    assert _rel(dx_m, dx_r) <= GRAD_RTOL
    for i, (a, b) in enumerate(zip(gp_m, gp_r)):
        assert (a is None) == (b is None), i
        if a is not None:
            assert _rel(a, b) <= GRAD_RTOL, names[i] if names else i
    for a, b in zip(gh_m, gh_r):
        assert (a is None) == (b is None)
        if a is not None:
            assert _rel(a, b) <= GRAD_RTOL


def _check_against_torch(kind, B, T, I, H, L, bi, lens=None, hx_grad=True, freeze=False):
    ref, mine = _models(kind, I, H, L, bi)
    if freeze:
        for m in (ref, mine):
            for p in m.parameters():
                p.requires_grad_(False)
    x, hx, wy, ws = _inputs(kind, B, T, I, H, L, bi)
    r = _run(ref, x, hx, wy, ws, "cpu", lens, hx_grad)
    m = _run(mine, x, hx, wy, ws, DEV, lens, hx_grad)
    _compare(m, r, [n for n, _ in ref.named_parameters()])


CASES = [
    # kind, B, T, I, H, L, bidirectional
    ("gru", 16, 24, 256, 256, 2, False),    # bs2
    ("gru", 64, 24, 256, 256, 2, False),    # bs4 (batch-paired)
    ("gru", 128, 24, 256, 256, 2, False),   # tc8, streamed projection
    ("gru", 160, 24, 256, 256, 2, False),   # tc8 after its GEMM (two waves)
    ("gru", 16, 20, 64, 256, 2, True),
    ("gru", 24, 20, 64, 128, 2, False),
    ("gru", 24, 20, 64, 128, 2, True),
    ("lstm", 16, 20, 64, 128, 2, False),
    ("lstm", 16, 20, 64, 128, 2, True),
    ("lstm", 24, 20, 64, 256, 2, False),
    ("lstm", 24, 20, 64, 256, 2, True),
    # batch not a multiple of the cluster's rows
    ("gru", 13, 16, 64, 256, 1, False),
    ("gru", 61, 16, 64, 256, 1, False),
    ("gru", 125, 16, 256, 256, 1, False),
    ("lstm", 7, 16, 64, 256, 1, True),
    ("gru", 11, 16, 64, 128, 1, True),
    # T = 1: no recurrent step inside the call, the whole dW_hh is the h_0 term
    ("gru", 16, 1, 64, 256, 2, True),
    ("gru", 128, 1, 256, 256, 2, False),
    ("lstm", 16, 1, 64, 128, 2, True),
    # wide-batch fallbacks (several waves)
    ("gru", 300, 4, 32, 128, 1, False),
    ("lstm", 152, 4, 32, 256, 1, False),
    ("lstm", 300, 4, 32, 128, 1, False),
]


@pytest.mark.parametrize("kind,B,T,I,H,L,bi", CASES)
def test_initial_state_matches_torch_cpu(kind, B, T, I, H, L, bi):
    _check_against_torch(kind, B, T, I, H, L, bi)


def _lengths(B, T, skew, seed=0):
    g = torch.Generator().manual_seed(seed)
    if skew == "one_long":
        lens = torch.randint(1, max(2, T // 4) + 1, (B,), generator=g)
        lens[B // 2] = T
    else:
        lens = 1 + (torch.arange(B) * (T - 1)) // max(B - 1, 1)
    return lens


PACKED = [
    ("gru", 16, 40, 256, 256, 2, False),
    ("gru", 64, 40, 256, 256, 2, False),
    ("gru", 128, 40, 256, 256, 2, False),
    ("gru", 16, 40, 64, 256, 2, True),      # reverse direction: the first real step t = len_b - 1 reads h_0
    ("gru", 24, 30, 64, 128, 1, True),
    ("lstm", 64, 30, 256, 128, 2, True),
    ("lstm", 64, 30, 256, 256, 2, True),
    ("gru", 300, 6, 32, 128, 1, True),      # wide-batch fallback, ragged
]


@pytest.mark.parametrize("skew", ["one_long", "rising"])
@pytest.mark.parametrize("kind,B,T,I,H,L,bi", PACKED)
def test_packed_initial_state_matches_torch_cpu(kind, B, T, I, H, L, bi, skew):
    _check_against_torch(kind, B, T, I, H, L, bi, lens=_lengths(B, T, skew))


@pytest.mark.parametrize("kind,B,bi", [("gru", 128, False), ("gru", 16, True), ("lstm", 24, True)])
def test_hx_without_grad_and_frozen_weights(kind, B, bi):
    """hx that does not require grad (weights trainable: no dh_0 is computed), and hx that does with every weight
    frozen (only dx and dh_0 / dc_0)."""
    H = 256
    _check_against_torch(kind, B, 20, 64, H, 2, bi, hx_grad=False)
    _check_against_torch(kind, B, 20, 64, H, 2, bi, freeze=True)


def _chunked(model, x, hx, chunks):
    """run x [B,T,I] as consecutive chunks that chain h_n -> hx without detach; returns y, h_n"""
    ys, h = [], hx
    for c in chunks:
        y, h = model(x[:, c], h)
        ys.append(y)
    return torch.cat(ys, dim=1), h


@pytest.mark.parametrize("B,tf32", [(16, False), (128, False), (128, True)])
def test_chunked_equals_whole(B, tf32):
    """T = 120 as 4 chunks of 30, and as 120 calls of one step, chaining the state without detach: outputs and states
    within 1e-6 of one whole call, dx and every parameter gradient within the gradient tolerance. Under TF32 mode the
    tc8 recurrence rounds the staged state; the staged h_0 must be rounded the same way (the forward is checked to the
    same 1e-6). The gradients are then single-pass TF32 GEMMs on both sides, but of other shapes (a one-step call's
    dW_hh is its exact fp32 h_0 term alone, the whole call's one TF32 contraction over T*B rows), so they agree to
    TF32's rounding (~2^-11 relative per operand; tests/test_gpu_tf32_mode.py sees ~1e-3 against fp64), not to 1e-4."""
    T, I, H = 120, 256, 256
    _, mine = _models("gru", I, H, 2, False, seed=4)
    g = torch.Generator().manual_seed(4)
    x0 = torch.randn(B, T, I, generator=g).to(DEV)
    h0 = (0.5 * torch.randn(2, B, H, generator=g)).to(DEV)
    wy = torch.randn(B, T, H, generator=g).to(DEV)
    wh = torch.randn(2, B, H, generator=g).to(DEV)
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32" if tf32 else "ieee"
    try:
        def run(chunks):
            mine.zero_grad(set_to_none=True)
            x = x0.clone().requires_grad_(True)
            h = h0.clone().requires_grad_(True)
            if chunks is None:
                y, hn = mine(x, h)
            else:
                y, hn = _chunked(mine, x, h, chunks)
            ((y * wy).sum() + (hn * wh).sum()).backward()
            return y.detach(), hn.detach(), x.grad, h.grad, [p.grad.clone() for p in mine.parameters()]

        whole = run(None)
        for name, chunks in (("4x30", [slice(i, i + 30) for i in range(0, T, 30)]),
                             ("120x1", [slice(i, i + 1) for i in range(T)])):
            got = run(chunks)
            bitwise = torch.equal(got[0], whole[0]) and torch.equal(got[1], whole[1])
            print(f"chunked {name} B={B} tf32={tf32}: outputs/states bit-identical to the whole call: {bitwise}; "
                  f"max |dy| {(got[0] - whole[0]).abs().max().item():.3g}")
            assert (got[0] - whole[0]).abs().max().item() <= 1e-6, name
            assert (got[1] - whole[1]).abs().max().item() <= 1e-6, name
            grad_err = max(_rel(a, b) for a, b in zip([got[2], got[3]] + got[4], [whole[2], whole[3]] + whole[4]))
            print(f"chunked {name} B={B} tf32={tf32}: gradients {grad_err:.3g} relative to the whole call")
            assert grad_err <= (TF32_GRAD_RTOL if tf32 else GRAD_RTOL), name
    finally:
        torch.backends.cuda.matmul.fp32_precision = saved


@pytest.mark.parametrize("kind,B,bi,packed", [("gru", 128, False, False), ("gru", 16, True, True),
                                              ("lstm", 24, True, False), ("lstm", 64, True, True)])
def test_zero_hx_is_bit_identical_to_none(kind, B, bi, packed):
    """hx = zeros (requiring grad, so dh_0 and the h_0 dW_hh term run) changes no output, state or gradient by a bit."""
    T, I, H, L = 30, 64, 256, 2
    _, mine = _models(kind, I, H, L, bi)
    x, hx, wy, ws = _inputs(kind, B, T, I, H, L, bi)
    lens = _lengths(B, T, "one_long") if packed else None

    def run(zero_hx):
        mine.zero_grad(set_to_none=True)
        xx = x.clone().to(DEV).requires_grad_(True)
        inp = xx if lens is None else pack_padded_sequence(xx, lens, batch_first=True, enforce_sorted=False)
        h0 = [torch.zeros_like(h, device=DEV).requires_grad_(True) for h in hx] if zero_hx else None
        out = mine(inp, None if h0 is None else (h0[0] if len(h0) == 1 else tuple(h0)))
        y = out[0] if lens is None else pad_packed_sequence(out[0], batch_first=True, total_length=T)[0]
        loss = (y * wy.to(DEV)).sum()
        for s, w in zip(_states(out), ws):
            loss = loss + (s * w.to(DEV)).sum()
        loss.backward()
        return [y.detach(), *[s.detach() for s in _states(out)], xx.grad] + [p.grad for p in mine.parameters()]

    for a, b in zip(run(True), run(False)):
        assert torch.equal(a, b)


def test_cuda_graph_replay_equals_eager():
    """Forward + backward with a static hx captured in a CUDA graph and replayed give the eager results."""
    B, T, I, H = 64, 20, 128, 256
    _, mine = _models("gru", I, H, 2, False)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, T, I, generator=g).to(DEV)
    h0 = (0.5 * torch.randn(2, B, H, generator=g)).to(DEV).requires_grad_(True)
    wy = torch.randn(B, T, H, generator=g).to(DEV)
    wh = torch.randn(2, B, H, generator=g).to(DEV)

    def step():
        y, hn = mine(x, h0)
        ((y * wy).sum() + (hn * wh).sum()).backward()
        return y.detach(), hn.detach()   # no autograd graph outlives the step (its nodes are bound to their stream)

    mine.zero_grad(set_to_none=True)
    h0.grad = None
    eager = [*(t.clone() for t in step()), h0.grad.clone()] + [p.grad.clone() for p in mine.parameters()]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            mine.zero_grad(set_to_none=True)
            h0.grad = None
            step()
    torch.cuda.current_stream().wait_stream(s)
    mine.zero_grad(set_to_none=True)
    h0.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_g, hn_g = step()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    got = [y_g, hn_g, h0.grad] + [p.grad for p in mine.parameters()]
    for a, b in zip(got, eager):
        assert torch.equal(a, b)


def test_runs_with_hx_are_bitwise_deterministic():
    for kind, B, T, I, H, bi, packed in (("gru", 128, 40, 256, 256, False, False), ("gru", 16, 40, 64, 256, True, True),
                                         ("lstm", 64, 30, 256, 256, True, False)):
        _, mine = _models(kind, I, H, 2, bi)
        x, hx, wy, ws = _inputs(kind, B, T, I, H, 2, bi)
        lens = _lengths(B, T, "one_long") if packed else None
        r1 = _run(mine, x, hx, wy, ws, DEV, lens)
        for _ in range(2):
            r2 = _run(mine, x, hx, wy, ws, DEV, lens)
            assert torch.equal(r1[0], r2[0]) and torch.equal(r1[2], r2[2]), kind
            for a, b in zip(r1[1] + r1[3] + r1[4], r2[1] + r2[3] + r2[4]):
                assert torch.equal(a, b), kind


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("batch_first", [False, True])
@pytest.mark.parametrize("with_hx", [False, True])
def test_unbatched_input_matches_torch(kind, batch_first, with_hx):
    """[T, I] input with an optional [L*D, H] state runs as one batch row and comes back unbatched (batch_first does
    not apply), as torch runs it."""
    import b200rnn

    T, I, H, L = 9, 32, 128, 2
    torch.manual_seed(2)
    cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    ref = cls(I, H, num_layers=L, bidirectional=True, batch_first=batch_first)
    mine = b200rnn.from_torch(ref).to(DEV)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(T, I, generator=g)
    hx = [torch.randn(2 * L, H, generator=g) for _ in range(1 if kind == "gru" else 2)] if with_hx else None

    def run(model, dev):
        xx = x.clone().to(dev).requires_grad_(True)
        h = None if hx is None else [t.clone().to(dev).requires_grad_(True) for t in hx]
        out = model(xx, None if h is None else (h[0] if kind == "gru" else tuple(h)))
        loss = out[0].square().sum() + sum(s.sum() for s in _states(out))
        loss.backward()
        values = [out[0].detach().cpu(), *[s.detach().cpu() for s in _states(out)]]
        grads = [xx.grad.cpu()] + ([t.grad.cpu() for t in h] if h is not None else [])
        return values, grads

    (v_r, g_r), (v_m, g_m) = run(ref, "cpu"), run(mine, DEV)
    assert [t.shape for t in v_m + g_m] == [t.shape for t in v_r + g_r]
    for a, b in zip(v_m, v_r):
        assert (a - b).abs().max().item() <= OUT_TOL
    for a, b in zip(g_m, g_r):
        assert _rel(a, b) <= GRAD_RTOL
