"""LSTM with projections (``proj_size``): ``b200rnn.LSTM(..., proj_size=P)`` against stock ``torch.nn.LSTM`` on CPU.

Tolerances as tests/test_gpu_initial_state.py: outputs and states 1e-5 absolute, gradients (every parameter including
``weight_hr``, dx, dh_0, dc_0) 1e-4 relative to the largest entry. The loss covers y, h_n and c_n. Every (H, P) runs
both its fixed-length and its ragged (VL) instantiation; B = 300 needs several waves of clusters for both widths."""
import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OUT_TOL = 1e-5
GRAD_RTOL = 1e-4
SIZES = [(128, 32), (128, 64), (256, 64), (256, 128)]


def _models(H, P, L, bi, I=40, batch_first=True, dropout=0.0, seed=0):
    import b200rnn

    torch.manual_seed(seed)
    ref = torch.nn.LSTM(I, H, num_layers=L, bidirectional=bi, batch_first=batch_first, proj_size=P, dropout=dropout)
    return ref, b200rnn.from_torch(ref).to(DEV)


def _inputs(B, T, I, H, P, L, D, batch_first=True, seed=11):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, I, generator=g) if batch_first else torch.randn(T, B, I, generator=g)
    hx = (0.5 * torch.randn(L * D, B, P, generator=g), 0.5 * torch.randn(L * D, B, H, generator=g))
    wy = torch.randn(*x.shape[:2], D * P, generator=g)
    ws = (torch.randn(L * D, B, P, generator=g), torch.randn(L * D, B, H, generator=g))
    return x, hx, wy, ws


def _run(model, x, wy, ws, dev, hx=None, lens=None, batch_first=True):
    """padded output, (h_n, c_n), dx, parameter gradients and hx gradients of sum(y * wy) + sum(state * ws)"""
    model.zero_grad(set_to_none=True)
    xx = x.clone().to(dev).requires_grad_(True)
    h0 = None if hx is None else tuple(h.clone().to(dev).requires_grad_(True) for h in hx)
    inp = xx if lens is None else pack_padded_sequence(xx, lens, batch_first=batch_first, enforce_sorted=False)
    y, states = model(inp, h0)
    if lens is not None:
        y = pad_packed_sequence(y, batch_first=batch_first, total_length=x.shape[1 if batch_first else 0])[0]
    loss = (y * wy.to(dev)).sum()
    for s, w in zip(states, ws):
        loss = loss + (s * w.to(dev)).sum()
    loss.backward()
    cpu = lambda t: None if t is None else t.detach().cpu()  # noqa: E731
    return (cpu(y), [cpu(s) for s in states], cpu(xx.grad), [cpu(p.grad) for p in model.parameters()],
            [] if h0 is None else [cpu(h.grad) for h in h0])


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _compare(mine, ref, what=""):
    y, st, dx, gp, gh = mine
    ry, rst, rdx, rgp, rgh = ref
    assert (y - ry).abs().max().item() <= OUT_TOL, what
    for a, b in zip(st, rst):
        assert (a - b).abs().max().item() <= OUT_TOL, what
    assert _rel(dx, rdx) <= GRAD_RTOL, what
    assert len(gp) == len(rgp)
    for i, (a, b) in enumerate(zip(gp, rgp)):
        assert _rel(a, b) <= GRAD_RTOL, (what, i)
    for a, b in zip(gh, rgh):
        assert _rel(a, b) <= GRAD_RTOL, what


@pytest.mark.parametrize("H,P", SIZES)
@pytest.mark.parametrize("L", [1, 2])
@pytest.mark.parametrize("bi", [False, True])
@pytest.mark.parametrize("batch_first", [True, False])
def test_projected_lstm_matches_torch_cpu(H, P, L, bi, batch_first):
    D = 2 if bi else 1
    ref, mine = _models(H, P, L, bi, batch_first=batch_first)
    x, _, wy, ws = _inputs(5, 9, 40, H, P, L, D, batch_first=batch_first)
    _compare(_run(mine, x, wy, ws, DEV, batch_first=batch_first), _run(ref, x, wy, ws, "cpu", batch_first=batch_first))


@pytest.mark.parametrize("H,P", [(128, 32), (256, 128)])
@pytest.mark.parametrize("B", [1, 7, 300])
def test_batch_sizes_including_several_waves(H, P, B):
    ref, mine = _models(H, P, 1, True)
    x, _, wy, ws = _inputs(B, 6, 40, H, P, 1, 2)
    _compare(_run(mine, x, wy, ws, DEV), _run(ref, x, wy, ws, "cpu"), f"B={B}")


@pytest.mark.parametrize("H,P", SIZES)
def test_initial_state_and_its_gradients(H, P):
    ref, mine = _models(H, P, 2, True)
    x, hx, wy, ws = _inputs(6, 8, 40, H, P, 2, 2)
    _compare(_run(mine, x, wy, ws, DEV, hx=hx), _run(ref, x, wy, ws, "cpu", hx=hx))


@pytest.mark.parametrize("H,P", SIZES)
def test_packed_sequence_skewed_lengths_padding_never_leaks(H, P):
    ref, mine = _models(H, P, 2, True)
    B, T = 11, 13
    x, hx, wy, ws = _inputs(B, T, 40, H, P, 2, 2)
    lens = torch.tensor([13, 1, 5, 13, 2, 9, 1, 7, 12, 3, 6])
    pad = torch.arange(T)[None, :] >= lens[:, None]
    x = x.masked_fill(pad[:, :, None], 0.0)
    wy = wy.masked_fill(pad[:, :, None], 0.0)
    a = _run(mine, x, wy, ws, DEV, hx=hx, lens=lens)
    _compare(a, _run(ref, x, wy, ws, "cpu", hx=hx, lens=lens))
    garbage = x.masked_fill(pad[:, :, None], 1e3)
    b = _run(mine, garbage, wy, ws, DEV, hx=hx, lens=lens)
    for u, v in zip([a[0], *a[1], *a[3], *a[4]], [b[0], *b[1], *b[3], *b[4]]):
        assert torch.equal(u, v)
    assert torch.equal(a[2].masked_fill(pad[:, :, None], 0), b[2].masked_fill(pad[:, :, None], 0))


@pytest.mark.parametrize("H,P", [(128, 64), (256, 64)])
def test_unbatched_input(H, P):
    ref, mine = _models(H, P, 2, True)
    x, hx, _, _ = _inputs(1, 7, 40, H, P, 2, 2)
    x, hx = x[0], tuple(h[:, 0] for h in hx)
    yr, (hr, cr) = ref(x, hx)
    with torch.no_grad():
        ym, (hm, cm) = mine(x.to(DEV), tuple(h.to(DEV) for h in hx))
    assert ym.shape == yr.shape == (7, 2 * P) and hm.shape == hr.shape == (4, P) and cm.shape == (4, H)
    for a, b in ((ym, yr), (hm, hr), (cm, cr)):
        assert (a.cpu() - b).abs().max().item() <= OUT_TOL


def test_bitwise_determinism_and_cuda_graph_replay():
    ref, mine = _models(256, 128, 2, True)
    x, hx, wy, ws = _inputs(9, 10, 40, 256, 128, 2, 2)
    a, b = _run(mine, x, wy, ws, DEV, hx=hx), _run(mine, x, wy, ws, DEV, hx=hx)
    for u, v in zip([a[0], *a[1], a[2], *a[3], *a[4]], [b[0], *b[1], b[2], *b[3], *b[4]]):
        assert torch.equal(u, v)

    mine.eval()
    xs = x.to(DEV)
    h0 = tuple(h.to(DEV) for h in hx)
    with torch.no_grad():
        eager = mine(xs, h0)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            mine(xs, h0)  # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            captured = mine(xs, h0)
        g.replay()
        torch.cuda.synchronize()
    assert torch.equal(eager[0], captured[0])
    assert torch.equal(eager[1][0], captured[1][0]) and torch.equal(eager[1][1], captured[1][1])


def test_dropout_masks_of_forward_and_backward_agree():
    """Train mode, p = 0.5, one step of one sequence: the units whose dW_ih_l1 column is zero are the ones the dropout
    zeroed. Layer 1 alone (stock torch) on h0 * mask / (1 - p) reproduces the output (forward mask), and autograd
    through the same mask reproduces dx (backward mask)."""
    import b200rnn

    p, H, P = 0.5, 256, 128
    torch.manual_seed(6)
    m = b200rnn.LSTM(64, H, num_layers=2, dropout=p, bidirectional=True, proj_size=P).to(DEV).train()
    layers = [torch.nn.LSTM(64 if i == 0 else 2 * P, H, bidirectional=True, proj_size=P) for i in range(2)]
    with torch.no_grad():
        for i, mod in enumerate(layers):
            for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh", "weight_hr"):
                for sfx in ("", "_reverse"):
                    getattr(mod, f"{n}_l0{sfx}").copy_(getattr(m, f"{n}_l{i}{sfx}").cpu())
    x = torch.randn(1, 1, 64)
    dy = torch.randn(1, 1, 2 * P)
    xm = x.to(DEV).requires_grad_(True)
    y, _ = m(xm)
    (y * dy.to(DEV)).sum().backward()
    kept = (m.weight_ih_l1.grad.abs().sum(0) != 0).cpu()
    frac = 1.0 - kept.float().mean().item()
    assert 0.3 < frac < 0.7, frac
    xr = x.clone().requires_grad_(True)
    h0 = layers[0](xr)[0]
    y_check = layers[1](h0 * kept / (1 - p))[0]
    (y_check * dy).sum().backward()
    assert (y.detach().cpu() - y_check.detach()).abs().max().item() <= OUT_TOL
    assert _rel(xm.grad.cpu(), xr.grad) <= GRAD_RTOL


def test_tf32_mode_within_tf32_bounds_of_float64():
    ref, mine = _models(256, 64, 2, True)
    x, hx, wy, ws = _inputs(6, 12, 40, 256, 64, 2, 2)
    old = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        got = _run(mine, x, wy, ws, DEV, hx=hx)
    finally:
        torch.backends.cuda.matmul.fp32_precision = old
    ref = ref.double()
    want = _run(ref, x.double(), wy.double(), tuple(w.double() for w in ws), "cpu", hx=tuple(h.double() for h in hx))
    assert (got[0].double() - want[0]).abs().max().item() <= 2e-3
    assert _rel(got[2].double(), want[2]) <= 5e-3
    for a, b in zip(got[3], want[3]):
        assert _rel(a.double(), b) <= 5e-3


def test_weight_hr_gradients_land_in_the_grad_bucket():
    from b200rnn.dp import GradBucket

    ref, mine = _models(128, 64, 2, True)
    bucket = GradBucket(mine)
    x, _, wy, ws = _inputs(4, 5, 40, 128, 64, 2, 2)
    names = [n for n, _ in mine.named_parameters()]
    assert names[4] == "weight_hr_l0" and names[9] == "weight_hr_l0_reverse"
    mine.zero_grad(set_to_none=False)
    y, (h, c) = mine(x.to(DEV))
    ((y * wy.to(DEV)).sum() + (h * ws[0].to(DEV)).sum() + (c * ws[1].to(DEV)).sum()).backward()
    yr, (hr, cr) = ref(x)
    ((yr * wy).sum() + (hr * ws[0]).sum() + (cr * ws[1]).sum()).backward()
    base = bucket.flat.data_ptr()
    for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters()):
        assert base <= p.grad.data_ptr() < base + bucket.nbytes, n
        assert _rel(p.grad.cpu(), q.grad) <= GRAD_RTOL, n
