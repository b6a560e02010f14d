"""Several models in one call (B200RNN_FLAG_MODELS, b200rnn/func.py) without a GPU: the descriptor's flag-gated fields,
what the library rejects, the workspace sizes for M models, the buffers the forward allocates for them, and the cases
that raise under torch.func transforms."""
import ctypes
import dataclasses

import pytest
import torch

from b200rnn import _lib
from b200rnn import func as bfunc
from b200rnn import functional as F

OK, ERR_INVALID, ERR_UNSUPPORTED = 0, -1, -2   # B200RNN_OK, B200RNN_ERR_INVALID, B200RNN_ERR_UNSUPPORTED


def _cfg(mode=_lib.GRU, H=64, L=2, D=2, batch_first=False, **kw):
    return F.RNNConfig(mode=mode, input_size=24, hidden_size=H, num_layers=L, num_dirs=D, dropout=0.25, training=True,
                       batch_first=batch_first, **kw)


def _desc(cfg, B=8, T=3, save=True, flags=0, models=None, strides=None):
    d = F._make_desc(cfg, B, T, save, model_strides=strides)
    d.flags |= flags
    if models is not None:
        d.models = models
    return d


def _ws(desc):
    lib = _lib.load()
    r, s = ctypes.c_size_t(0), ctypes.c_size_t(0)
    rc = lib.b200rnn_workspace_bytes(ctypes.byref(desc), ctypes.byref(r), ctypes.byref(s))
    return rc, r.value, s.value, lib.b200rnn_last_error().decode()


def test_model_fields_are_read_only_with_the_flag():
    one = _ws(_desc(_cfg()))
    assert one[0] == OK
    d = _desc(_cfg())
    d.models, d.model_strides = -7, None   # garbage without FLAG_MODELS
    assert _ws(d) == one
    d.models = 1
    d.flags |= _lib.FLAG_MODELS
    assert _ws(d) == one


@pytest.mark.parametrize("M", (0, -1))
def test_model_count_below_one_is_invalid(M):
    cfg = dataclasses.replace(_cfg(), models=3)
    rc, _, _, msg = _ws(_desc(cfg, models=M))
    assert rc == ERR_INVALID and "models must be >= 1" in msg


def test_several_models_without_strides_are_invalid():
    d = _desc(_cfg())
    d.flags |= _lib.FLAG_MODELS
    d.models = 2
    rc, _, _, msg = _ws(d)
    assert rc == ERR_INVALID and "model_strides" in msg


@pytest.mark.parametrize("what", ("proj", "f16", "bf16", "f32_params", "accumulate"))
def test_several_models_reject_what_they_do_not_run(what):
    kw, flags = {}, 0
    if what == "proj":
        kw = dict(mode=_lib.LSTM, H=128, proj_size=32)
    elif what in ("f16", "bf16"):
        kw = dict(dtype=torch.float16 if what == "f16" else torch.bfloat16)
    elif what == "f32_params":
        kw = dict(dtype=torch.float16, master_f32=True)
    else:
        flags = _lib.FLAG_ACCUMULATE_GRADS
    cfg = dataclasses.replace(_cfg(**kw), models=2)
    rc, _, _, msg = _ws(_desc(cfg, flags=flags))
    assert rc == ERR_UNSUPPORTED, (what, rc, msg)
    assert "several models in one call are float32 only" in msg
    assert _ws(_desc(dataclasses.replace(cfg, models=1), flags=flags))[0] == OK


def test_several_models_reject_ragged_lengths_and_the_shell_entry():
    lib = _lib.load()
    cfg = dataclasses.replace(_cfg(), models=2)
    d = _desc(cfg)
    fake = ctypes.c_void_p(256)   # never dereferenced: the call is refused before anything runs
    params = _lib.ptr_array([256] * 16)
    rc = lib.b200rnn_forward_hx(ctypes.byref(d), fake, 24 * 8, 24, params, fake, 0, 0, None, None, fake, None, fake,
                                fake, 0, 0, None, fake, None)
    assert rc == ERR_UNSUPPORTED and "take no lengths" in lib.b200rnn_last_error().decode()
    rc = lib.b200rnn_forward_fused(ctypes.byref(_desc(dataclasses.replace(cfg, mode=_lib.GRU), models=2)), fake, 0, 0,
                                   params, fake, 0, 0, fake, None, fake, fake, 0, 0, None, None, None, 0.0, None, None,
                                   None, None, None)
    assert rc == ERR_UNSUPPORTED


@pytest.mark.parametrize("mode,H", ((_lib.GRU, 64), (_lib.LSTM, 128), (_lib.RNN_TANH, 208)))
@pytest.mark.parametrize("save", (True, False))
def test_workspace_is_m_one_model_blocks(mode, H, save):
    cfg = _cfg(mode=mode, H=H)
    rc, r1, s1, _ = _ws(_desc(cfg, save=save))
    assert rc == OK
    for M in (2, 3, 8, 32):
        rc, r, s, _ = _ws(_desc(dataclasses.replace(cfg, models=M), save=save))
        assert rc == OK and (r, s) == (M * r1, M * s1), M
        assert r1 % 256 == 0 and s1 % 256 == 0   # each model's blocks stay 256-byte aligned


@pytest.mark.parametrize("mode", (_lib.GRU, _lib.LSTM, _lib.RNN_RELU))
@pytest.mark.parametrize("batch_first", (False, True))
@pytest.mark.parametrize("save", (True, False))
def test_forward_buffers_for_m_models(mode, batch_first, save):
    """the buffers of an M-model call are the one-model buffers with a leading [M], dense (what the library's model
    strides assume), on the meta device: host arithmetic only"""
    T, B, I, M = 3, 8, 24, 5
    cfg = _cfg(mode=mode, batch_first=batch_first)
    x1 = torch.empty(T, B, I, device="meta")
    _, r1, _, y1, ys1, h1, c1 = F._forward_buffers(x1, cfg, save, with_scratch=False)
    xm = torch.empty(M, T, B, I, device="meta")
    _, r, _, y, ys, h, c = F._forward_buffers(xm, dataclasses.replace(cfg, models=M), save, with_scratch=False)
    assert ys == ys1
    for one, many in ((r1, r), (y1, y), (h1, h), (c1, c)):
        if one is None:
            assert many is None
            continue
        assert many.shape == (M, *one.shape)
        assert many.is_contiguous() and many.stride()[1:] == one.stride()


def test_dx_buffer_of_m_models_is_dense():
    x = torch.empty(4, 6, 3, 24).transpose(1, 2)   # a batch-first x seen time-major, per model
    assert F._dx_buffer(x).is_contiguous()
    assert F._dx_buffer(torch.empty(6, 3, 24).expand(4, 6, 3, 24)).is_contiguous()


@pytest.mark.parametrize("case", ("proj", "f16", "autocast", "packed", "grad_sink"))
def test_out_of_scope_cases_raise_under_torch_func(case):
    cfg, lengths, sink = _cfg(), None, None
    if case == "proj":
        cfg = _cfg(mode=_lib.LSTM, H=128, proj_size=32)
    elif case == "f16":
        cfg = _cfg(dtype=torch.float16)
    elif case == "autocast":
        cfg = _cfg(dtype=torch.bfloat16, master_f32=True)
    elif case == "packed":
        lengths = torch.tensor([3, 2])
    else:
        sink = lambda ws: ws  # noqa: E731
    with pytest.raises(_lib.B200RNNError, match={"proj": "proj_size", "f16": "float32", "autocast": "autocast",
                                                 "packed": "PackedSequence", "grad_sink": "gradient sink"}[case]):
        bfunc.check_supported(cfg, lengths, sink)
    bfunc.check_supported(_cfg(), None, None)


def test_model_strides_follow_the_tensors():
    M = 3
    cfg = dataclasses.replace(_cfg(L=1, D=1), models=M, rng_stride=2)
    x = torch.empty(M, 5, 2, 24)
    shared = torch.empty(192, 64).expand(M, 192, 64)
    ws = [torch.empty(M, 192, 24), shared, torch.empty(M, 192), torch.empty(M, 192)]
    assert F._model_strides(cfg, x, ws) == [5 * 2 * 24, 2, 192 * 24, 0, 192, 192]
    assert F._model_strides(dataclasses.replace(cfg, models=1), x[0], [w[0] for w in ws]) is None
