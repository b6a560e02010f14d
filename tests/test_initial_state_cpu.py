"""The initial-state contract without a GPU: hx is checked as stock torch checks it (same exception types, and the same
messages for shapes), host tensors still fail loudly with a NotImplementedError, and the hx entry points of the C ABI
reject inconsistent state pointers before anything touches the device."""
import ctypes

import pytest
import torch

import b200rnn
from b200rnn import _lib

STOCK = {"gru": b200rnn.modules._TORCH_GRU, "lstm": b200rnn.modules._TORCH_LSTM}
MINE = {"gru": b200rnn.GRU, "lstm": b200rnn.LSTM}


def _pair(kind, **kw):
    torch.manual_seed(0)
    stock = STOCK[kind](8, 16, **kw)
    mine = MINE[kind](8, 16, **kw)
    return stock, mine


def _hx(kind, *shape, dtype=torch.float32, device="cpu"):
    h = torch.zeros(*shape, dtype=dtype, device=device)
    return h if kind == "gru" else (h, torch.zeros(*shape, dtype=dtype, device=device))


def _raised(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 - the exception itself is what is compared
        return e
    return None


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("case", [
    # (module kwargs, input shape, hx shape)
    (dict(num_layers=2), (5, 3, 8), (1, 3, 16)),                      # wrong layer count
    (dict(num_layers=1, bidirectional=True), (5, 3, 8), (1, 3, 16)),  # missing direction
    (dict(), (5, 3, 8), (1, 4, 16)),                                  # wrong batch
    (dict(batch_first=True), (3, 5, 8), (1, 5, 16)),                  # batch taken from the wrong dimension
    (dict(), (5, 3, 8), (1, 3, 15)),                                  # wrong hidden size
    (dict(), (5, 3, 8), (3, 16)),                                     # 2-D hx for 3-D input
    (dict(), (5, 8), (1, 1, 16)),                                     # 3-D hx for unbatched input
    (dict(num_layers=2), (5, 8), (1, 16)),                            # unbatched, wrong layer count
])
def test_hx_shape_errors_match_torch(kind, case):
    kw, xshape, hshape = case
    stock, mine = _pair(kind, **kw)
    x = torch.randn(*xshape)
    want = _raised(lambda: stock(x, _hx(kind, *hshape)))
    got = _raised(lambda: mine(x, _hx(kind, *hshape)))
    assert want is not None and got is not None
    assert type(got) is type(want) and str(got) == str(want)


def test_lstm_cell_state_shape_error_matches_torch():
    stock, mine = _pair("lstm")
    x = torch.randn(5, 3, 8)
    hx = (torch.zeros(1, 3, 16), torch.zeros(1, 2, 16))
    want, got = _raised(lambda: stock(x, hx)), _raised(lambda: mine(x, hx))
    assert type(got) is type(want) and str(got) == str(want) == "Expected hidden[1] size (1, 3, 16), got [1, 2, 16]"


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_hx_dtype_and_device_errors_are_runtime_errors(kind):
    """torch reports a state of another dtype or device from its kernels as RuntimeError; so does the drop-in, before
    the missing CPU path."""
    stock, mine = _pair(kind)
    x = torch.randn(5, 3, 8)
    want = _raised(lambda: stock(x, _hx(kind, 1, 3, 16, dtype=torch.float64)))
    got = _raised(lambda: mine(x, _hx(kind, 1, 3, 16, dtype=torch.float64)))
    assert isinstance(want, RuntimeError) and isinstance(got, RuntimeError)
    assert not isinstance(got, NotImplementedError) and "same dtype" in str(got)
    got = _raised(lambda: mine(x, _hx(kind, 1, 3, 16, device="meta")))
    assert isinstance(got, RuntimeError) and not isinstance(got, NotImplementedError) and "same device" in str(got)


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_host_tensors_with_hx_or_unbatched_raise_not_implemented(kind):
    """A valid hx or an unbatched input on the host reaches the missing CPU path: B200RNNError and NotImplementedError
    (torch's error for an operator without a kernel for the tensor's backend)."""
    _, mine = _pair(kind, num_layers=2)
    for args in ((torch.randn(5, 3, 8), _hx(kind, 2, 3, 16)), (torch.randn(5, 8),), (torch.randn(5, 8), _hx(kind, 2, 16))):
        e = _raised(lambda: mine(*args))
        assert isinstance(e, NotImplementedError) and isinstance(e, b200rnn.B200RNNError), args[0].shape
        assert "no CPU path" in str(e)


def test_input_rank_error_matches_torch():
    stock, mine = _pair("gru")
    x = torch.randn(2, 5, 3, 8)
    want, got = _raised(lambda: stock(x)), _raised(lambda: mine(x))
    assert type(got) is type(want) is ValueError and str(got) == str(want)


def test_packed_hx_shape_error_matches_torch():
    stock, mine = _pair("gru")
    packed = torch.nn.utils.rnn.pack_padded_sequence(torch.randn(4, 3, 8), torch.tensor([4, 2, 1]))
    want = _raised(lambda: stock(packed, torch.zeros(1, 2, 16)))
    got = _raised(lambda: mine(packed, torch.zeros(1, 2, 16)))
    assert type(got) is type(want) and str(got) == str(want)


# ---- C ABI -------------------------------------------------------------------------------------------------------

FAKE = ctypes.c_void_p(256)  # never dereferenced: every call below must fail in its argument checks


def _forward_hx(desc, h_0, c_0, x=None):
    lib = _lib.load()
    return lib.b200rnn_forward_hx(ctypes.byref(desc), x, 0, 0, None, None, 0, 0, h_0, c_0, None, None, None, None,
                                  0, 0, None, None, None)


def _backward_hx(desc, h_0, c_0, dh_0, dc_0, dy=None):
    lib = _lib.load()
    return lib.b200rnn_backward_hx(ctypes.byref(desc), None, 0, 0, None, None, 0, 0, dy, 0, 0, None, None,
                                   h_0, c_0, dh_0, dc_0, None, None, None, 0, 0, None, None, None)


def test_forward_hx_rejects_inconsistent_states_before_touching_the_device():
    lib = _lib.load()
    gru = _lib.Desc(_lib.GRU, 2, 2, 16, 128, 1, 1, 0, 0.0, 0)
    lstm = _lib.Desc(_lib.LSTM, 2, 2, 16, 128, 1, 1, 0, 0.0, 0)
    assert _forward_hx(gru, FAKE, FAKE) == -1 and b"no cell state" in lib.b200rnn_last_error()
    assert _forward_hx(lstm, None, FAKE) == -1 and b"c_0 without h_0" in lib.b200rnn_last_error()
    assert _forward_hx(lstm, FAKE, FAKE) == -1 and b"null pointer" in lib.b200rnn_last_error()
    assert _forward_hx(gru, FAKE, None) == -1 and b"null pointer" in lib.b200rnn_last_error()


def test_backward_hx_rejects_inconsistent_states_before_touching_the_device():
    lib = _lib.load()
    gru = _lib.Desc(_lib.GRU, 2, 2, 16, 128, 1, 1, 0, 0.0, 0)
    lstm = _lib.Desc(_lib.LSTM, 2, 2, 16, 128, 1, 1, 0, 0.0, 0)
    assert _backward_hx(gru, FAKE, None, None, FAKE, dy=FAKE) == -1 and b"no cell state" in lib.b200rnn_last_error()
    assert _backward_hx(gru, FAKE, FAKE, None, None, dy=FAKE) == -1 and b"no cell state" in lib.b200rnn_last_error()
    assert _backward_hx(lstm, None, FAKE, None, None, dy=FAKE) == -1 and b"c_0 without h_0" in lib.b200rnn_last_error()
    assert _backward_hx(lstm, FAKE, FAKE, FAKE, FAKE) == -1 and b"null pointer" in lib.b200rnn_last_error()
    assert _backward_hx(gru, FAKE, None, FAKE, None, dy=FAKE) == -1 and b"null pointer" in lib.b200rnn_last_error()


def test_abi_version_covers_the_hx_entry_points():
    assert _lib.ABI_VERSION == 4
    assert {"b200rnn_forward_hx", "b200rnn_backward_hx"} <= set(_lib.SYMBOLS)
