"""LSTM with projections (``proj_size``) without a GPU: the module surface matches stock ``torch.nn.LSTM(proj_size=P)``
(parameters, init, state_dict, pickling, exceptions and their messages), the C ABI validates the descriptor and sizes
the workspace for it, and a float64 LSTMP (forward and analytic BPTT, below) is pinned to torch's double-precision LSTM
to 1e-12."""
import ctypes
import io

import numpy as np
import pytest
import torch

import b200rnn
from b200rnn import _lib

STOCK_LSTM = b200rnn.modules._TORCH_LSTM
STOCK_GRU = b200rnn.modules._TORCH_GRU
SUPPORTED = [(128, 32), (128, 64), (256, 64), (256, 128)]


def _raised(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 - the exception itself is what is compared
        return e
    return None


# ---- module surface ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,P", SUPPORTED)
@pytest.mark.parametrize("bi", [False, True])
def test_parameters_match_stock_names_order_shapes_and_init(H, P, bi):
    stock = STOCK_LSTM(24, H, num_layers=2, bidirectional=bi, proj_size=P)
    mine = b200rnn.LSTM(24, H, num_layers=2, bidirectional=bi, proj_size=P)
    assert [(n, p.shape) for n, p in mine.named_parameters()] == [(n, p.shape) for n, p in stock.named_parameters()]
    assert mine.proj_size == P and repr(mine) == repr(stock)
    bound = 1.0 / H ** 0.5
    for n, p in mine.named_parameters():
        assert p.abs().max().item() <= bound and p.std().item() > 0.3 * bound, n
    assert [len(w) for w in mine.all_weights] == [len(w) for w in stock.all_weights] == [5] * (4 if bi else 2)


def test_state_dict_round_trips_pickles_and_from_torch():
    stock = STOCK_LSTM(24, 256, num_layers=2, bidirectional=True, proj_size=128, batch_first=True)
    mine = b200rnn.LSTM(24, 256, num_layers=2, bidirectional=True, proj_size=128, batch_first=True)
    mine.load_state_dict(stock.state_dict())
    back = STOCK_LSTM(24, 256, num_layers=2, bidirectional=True, proj_size=128, batch_first=True)
    back.load_state_dict(mine.state_dict())
    for (n, a), (_, b) in zip(stock.state_dict().items(), back.state_dict().items()):
        assert torch.equal(a, b), n
    buf = io.BytesIO()
    torch.save(mine, buf)
    buf.seek(0)
    again = torch.load(buf, weights_only=False)
    assert again.proj_size == 128 and torch.equal(again.weight_hr_l1_reverse, mine.weight_hr_l1_reverse)
    twin = b200rnn.from_torch(stock)
    assert isinstance(twin, b200rnn.LSTM) and twin.proj_size == 128
    assert torch.equal(twin.weight_hr_l0, stock.weight_hr_l0)


@pytest.mark.parametrize("kw", [dict(proj_size=-1), dict(proj_size=128), dict(proj_size=200)])
def test_value_errors_match_torch(kw):
    a, b = _raised(lambda: STOCK_LSTM(8, 128, **kw)), _raised(lambda: b200rnn.LSTM(8, 128, **kw))
    assert type(a) is type(b) is ValueError and str(a) == str(b)


def test_gru_with_proj_size_raises_torchs_value_error():
    a, b = _raised(lambda: STOCK_GRU(8, 128, proj_size=4)), _raised(lambda: b200rnn.GRU(8, 128, proj_size=4))
    assert type(a) is type(b) is ValueError and str(a) == str(b)
    b200rnn.GRU(8, 128, proj_size=0)  # what from_torch passes for a GRU


@pytest.mark.parametrize("H,P", [(128, 4), (128, 48), (128, 96), (256, 32), (256, 100), (64, 16), (512, 128)])
def test_unsupported_projection_sizes_raise_not_implemented(H, P):
    with pytest.raises(NotImplementedError, match="proj_size 32 or 64.*proj_size 64 or 128"):
        b200rnn.LSTM(8, H, proj_size=P)


@pytest.mark.parametrize("case", [
    # (module kwargs, input shape, h_0 shape, c_0 shape)
    (dict(num_layers=2), (5, 3, 8), (2, 3, 128), (2, 3, 128)),          # h_0 carries H, not P
    (dict(num_layers=2), (5, 3, 8), (2, 3, 32), (2, 3, 32)),            # c_0 carries P, not H
    (dict(bidirectional=True), (5, 3, 8), (1, 3, 32), (2, 3, 128)),     # missing direction
    (dict(batch_first=True), (5, 3, 8), (1, 3, 32), (1, 3, 128)),       # batch taken from dim 0
    (dict(), (5, 8), (1, 2, 32), (1, 2, 128)),                          # unbatched input, batched state
])
def test_hx_shape_errors_match_torch(case):
    kw, xs, hs, cs = case
    torch.manual_seed(0)
    stock, mine = STOCK_LSTM(8, 128, proj_size=32, **kw), b200rnn.LSTM(8, 128, proj_size=32, **kw)
    x, hx = torch.zeros(*xs), (torch.zeros(*hs), torch.zeros(*cs))
    a, b = _raised(lambda: stock(x, hx)), _raised(lambda: mine(x, hx))
    assert a is not None and type(a) is type(b) and str(a) == str(b)


# ---- C ABI -------------------------------------------------------------------------------------------------------
def _desc(mode=_lib.LSTM, B=3, T=5, I=16, H=128, L=2, D=2, training=1, p=0.25, P=32):
    return _lib.Desc(mode, B, T, I, H, L, D, training, p, _lib.FLAG_PROJ if P else 0, P)


def _ws(desc):
    r, s = ctypes.c_size_t(0), ctypes.c_size_t(0)
    rc = _lib.load().b200rnn_workspace_bytes(ctypes.byref(desc), ctypes.byref(r), ctypes.byref(s))
    return rc, r.value, s.value


def test_proj_size_is_read_only_with_its_flag():
    """A descriptor that ends at `flags` (written before proj_size existed) means no projection, whatever memory
    follows it: the library reads proj_size only under B200RNN_FLAG_PROJ, so the ABI version stays 4."""
    assert _lib.ABI_VERSION == 4 and _lib.load().b200rnn_version() == 4
    assert _lib.Desc(0, 1, 1, 1, 128, 1, 1, 0, 0.0, 0).proj_size == 0  # positional: no projection
    unflagged = _desc(P=0)
    unflagged.proj_size = 12345  # stands for whatever follows a ten-field descriptor
    plain = _ws(_desc(P=0))
    assert _ws(unflagged) == plain and plain[0] == 0
    assert _ws(_desc(P=32))[1] > plain[1]  # flagged: the reserve adds m [T,B,H] per (layer, direction)


def test_descriptor_validation():
    lib = _lib.load()
    for kw in (dict(P=-1), dict(P=128), dict(P=256), dict(mode=_lib.GRU, P=32)):
        assert _ws(_desc(**kw))[0] == -1, kw
        assert b"proj_size" in lib.b200rnn_last_error()
    for kw in (dict(P=48), dict(H=256, P=32), dict(P=16)):
        assert _ws(_desc(**kw))[0] == -2, kw
        assert b"hidden_size/4 and hidden_size/2" in lib.b200rnn_last_error()
    for H, P in SUPPORTED:
        assert _ws(_desc(H=H, P=P))[0] == 0
    n = ctypes.c_size_t(0)
    assert lib.b200rnn_wcache_bytes(ctypes.byref(_desc()), ctypes.byref(n)) == -2


def test_fused_entry_points_refuse_a_projected_descriptor():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    params = _lib.ptr_array([256] * 20)
    d = _desc()
    rc = lib.b200rnn_forward_fused(ctypes.byref(d), fake, 0, 0, params, fake, 0, 0, fake, fake, None, fake, 0, 0,
                                   None, None, None, 0.0, None, None, None, None, None)
    assert rc == -2 and b"proj_size" in lib.b200rnn_last_error()
    rc = lib.b200rnn_backward_fused(ctypes.byref(d), fake, 0, 0, params, fake, 0, 0, fake, 0, 0, None, 0.0, None, None,
                                    fake, fake, None, 0, 0, params, None, None, 0.0, None, None, None)
    assert rc == -2 and b"proj_size" in lib.b200rnn_last_error()


@pytest.mark.parametrize("H,P", SUPPORTED)
@pytest.mark.parametrize("L,D,p", [(1, 1, 0.0), (2, 2, 0.25), (3, 1, 0.0)])
def test_reserve_follows_the_formula(H, P, L, D, p):
    """reserve = header + per (layer, dir): gates [TB,4H], c [TB,H], m [TB,H]; per inner layer: output [TB,D*P] and,
    with dropout, its dropped copy; then one alignment pad. Every block is rounded up to 64 floats."""
    B, T = 3, 5
    al = lambda n: (n + 63) // 64 * 64  # noqa: E731
    TB = T * B
    floats = 64 + L * D * (al(TB * 4 * H) + 2 * al(TB * H)) + (L - 1) * al(TB * D * P) * (2 if p > 0 else 1) + 64
    rc, r, s = _ws(_desc(B=B, T=T, H=H, L=L, D=D, p=p, P=P))
    assert rc == 0 and r == floats * 4
    rc0, r0, s0 = _ws(_desc(B=B, T=T, H=H, L=L, D=D, p=p, P=0))
    assert rc0 == 0 and s >= TB * P * D * 4  # scratch holds dh [T,B,P] per direction


# ---- float64 oracle ----------------------------------------------------------------------------------------------
def _sig(v):
    return 1.0 / (1.0 + np.exp(-v))


def lstmp_layer_forward(x, w_ih, w_hh, b_ih, b_hh, w_hr, h0, c0, reverse=False):
    """One direction of one LSTMP layer in float64: x [T,B,I] -> y [T,B,P], h_T, c_T and what the backward needs."""
    T = x.shape[0]
    H = w_hh.shape[0] // 4
    h, c = h0, c0
    y = np.zeros((T, x.shape[1], w_hr.shape[0]))
    cache = []
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        a = x[t] @ w_ih.T + b_ih + h @ w_hh.T + b_hh
        i, f, g, o = _sig(a[:, :H]), _sig(a[:, H:2 * H]), np.tanh(a[:, 2 * H:3 * H]), _sig(a[:, 3 * H:])
        c_new = f * c + i * g
        m = o * np.tanh(c_new)
        cache.append((t, h, c, i, f, g, o, c_new, m))
        h, c = m @ w_hr.T, c_new
        y[t] = h
    return y, h, c, cache


def lstmp_layer_backward(x, w_ih, w_hh, w_hr, cache, dy, dh_T, dc_T):
    """Analytic BPTT of lstmp_layer_forward: dx, dW_ih, dW_hh, db (= db_ih = db_hh), dW_hr, dh_0, dc_0."""
    dx = np.zeros_like(x)
    dw_ih, dw_hh, dw_hr = np.zeros_like(w_ih), np.zeros_like(w_hh), np.zeros_like(w_hr)
    db = np.zeros(w_ih.shape[0])
    dh, dc = dh_T.copy(), dc_T.copy()
    for t, h_prev, c_prev, i, f, g, o, c_new, m in reversed(cache):
        dh = dh + dy[t]
        dw_hr += dh.T @ m
        dm = dh @ w_hr
        tc = np.tanh(c_new)
        do = dm * tc
        dc = dc + dm * o * (1 - tc * tc)
        da = np.concatenate([dc * g * i * (1 - i), dc * c_prev * f * (1 - f), dc * i * (1 - g * g), do * o * (1 - o)], 1)
        dc = dc * f
        dx[t] = da @ w_ih
        dw_ih += da.T @ x[t]
        dw_hh += da.T @ h_prev
        db += da.sum(0)
        dh = da @ w_hh
    return dx, dw_ih, dw_hh, db, dw_hr, dh, dc


def lstmp_forward_backward(x, weights, L, D, h0, c0, dy, dh_n, dc_n):
    """Multi-layer (bi)LSTMP without dropout: outputs, final states and every gradient, in float64."""
    layer_in, caches, hn, cn = [x], [], np.zeros_like(h0), np.zeros_like(c0)
    for l in range(L):
        outs = []
        for d in range(D):
            k = l * D + d
            w = weights[5 * k:5 * k + 5]
            y, hn[k], cn[k], cache = lstmp_layer_forward(layer_in[-1], *w, h0[k], c0[k], reverse=d == 1)
            outs.append(y)
            caches.append(cache)
        layer_in.append(np.concatenate(outs, 2))
    grads = [None] * len(weights)
    dh0, dc0 = np.zeros_like(h0), np.zeros_like(c0)
    dout = dy
    P = h0.shape[2]
    for l in range(L - 1, -1, -1):
        din = np.zeros_like(layer_in[l])
        for d in range(D):
            k = l * D + d
            w_ih, w_hh, _, _, w_hr = weights[5 * k:5 * k + 5]
            dx, dwi, dwh, db, dwr, dh0[k], dc0[k] = lstmp_layer_backward(
                layer_in[l], w_ih, w_hh, w_hr, caches[k], dout[:, :, d * P:(d + 1) * P], dh_n[k], dc_n[k])
            din += dx
            grads[5 * k:5 * k + 5] = [dwi, dwh, db, db, dwr]
        dout = din
    return layer_in[-1], hn, cn, dout, grads, dh0, dc0


@pytest.mark.parametrize("H,P,L,bi", [(16, 4, 1, False), (16, 8, 2, True), (12, 3, 3, False)])
def test_float64_oracle_matches_torch_double(H, P, L, bi):
    D = 2 if bi else 1
    T, B, I = 6, 3, 5
    torch.manual_seed(3)
    ref = STOCK_LSTM(I, H, num_layers=L, bidirectional=bi, proj_size=P).double()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(T, B, I, generator=g, dtype=torch.float64, requires_grad=True)
    h0 = torch.randn(L * D, B, P, generator=g, dtype=torch.float64, requires_grad=True)
    c0 = torch.randn(L * D, B, H, generator=g, dtype=torch.float64, requires_grad=True)
    dy = torch.randn(T, B, D * P, generator=g, dtype=torch.float64)
    dhn = torch.randn(L * D, B, P, generator=g, dtype=torch.float64)
    dcn = torch.randn(L * D, B, H, generator=g, dtype=torch.float64)
    y, (hn, cn) = ref(x, (h0, c0))
    ((y * dy).sum() + (hn * dhn).sum() + (cn * dcn).sum()).backward()
    w = [p.detach().numpy() for p in ref.parameters()]
    oy, ohn, ocn, odx, og, odh0, odc0 = lstmp_forward_backward(
        x.detach().numpy(), w, L, D, h0.detach().numpy(), c0.detach().numpy(), dy.numpy(), dhn.numpy(), dcn.numpy())
    close = lambda a, b: np.abs(a - b.detach().numpy()).max() <= 1e-12 * max(1.0, np.abs(a).max())  # noqa: E731
    assert close(oy, y) and close(ohn, hn) and close(ocn, cn)
    assert close(odx, x.grad) and close(odh0, h0.grad) and close(odc0, c0.grad)
    for a, p in zip(og, ref.parameters()):
        assert close(a, p.grad)
