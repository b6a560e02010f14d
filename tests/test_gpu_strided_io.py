"""Sequence tensors as callers lay them out: offset, gapped, broadcast and size-1 x / dy / y / dx.

``rnn_forward`` takes x with any strides (only a feature stride other than 1 is copied), and the C ABI lets direct
callers stride y, dy and dx too. Each route that reads or writes them decides on its own whether it can use the
layout in place: the fp32 input projection's 3-D TMA map or the gather copy, the FFMA GEMM's vector or scalar loads,
the 16-bit map or copy16, widen16 / narrow16, the LayerNorm prologue, valid_rows for ragged batches, and the scalar y /
dy accesses of the recurrence kernels. Every case here runs the same call on the view and on a dense copy of it (same
weights, same dropout state) and asserts bitwise equal results wherever both run the same GEMM math; the C ABI cases
whose dx alignment moves the dgrad GEMM from the tensor cores to FFMA are held to the float64 bound of
test_gpu_numerics_f64.py instead. test_routes runs the catalogue under B200RNN_DEBUG and checks that each layout takes
the route it is meant to, so the matrix cannot quietly collapse onto the dense path.

Every view lies inside a buffer covering its whole footprint plus a margin, so no access, right or wrong, leaves the
allocation."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from test_gpu_numerics_f64 import _norm_err, _run_torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
MARGIN = 256
SENTINEL = 0xFFA1B2C3 - (1 << 32)   # a NaN pattern no kernel writes, as int32
SENTINEL16 = 0xB2C3 - (1 << 16)     # its low half, for 16-bit buffers


# ---- layouts --------------------------------------------------------------------------------------------------------

def x_layout(name, T, B, I):
    """(size, stride, storage offset) of a time-major [T,B,I] view of layout `name` (size-1 layouts change T or B)"""
    P = I + 8
    return {
        "dense": ((T, B, I), (B * I, I, 1), 0),
        "pad8": ((T, B, I), (B * P, P, 1), 0),                    # feats[..., :I] of a row of I + 8
        "off1": ((T, B, I), (B * P, P, 1), 1),                    # feats[..., 1:1+I]: misaligned base, odd row stride
        "off3": ((T, B, I), (B * P, P, 1), 3),
        "bgap": ((T, B, I), (2 * B * I, 2 * I, 1), 0),            # base[:, ::2]
        "bsub": ((T, B, I), (2 * B * I, I, 1), 0),                # base[:, :B] of a 2B batch
        "tgap": ((T, B, I), (2 * B * P, P, 1), 8),                # base[::2, :, 8:8+I]
        "bcast_b": ((T, B, I), (I, 0, 1), 0),                     # one sequence in every row
        "bcast_t": ((T, B, I), (0, I, 1), 0),                     # one step repeated over time
        "b1": ((T, 1, I), (I, 1, 1), 0),                          # B = 1 with batch stride 1
        "t1": ((1, B, I), (3, I, 1), 0),                          # T = 1 with time stride 3
    }[name]


def backing(size, stride, off):
    """elements of a buffer that holds the view and, from its first element on, its dense footprint, plus MARGIN: an
    access through a wrong stride or a dense-layout assumption stays inside it"""
    foot = off + sum((n - 1) * s for n, s in zip(size, stride)) + 1
    numel = 1
    for n in size:
        numel *= n
    return max(foot, off + numel) + MARGIN


def backed(size, stride, off, dtype, seed):
    """as_strided view on a fresh randn buffer (see backing)"""
    buf = torch.randn(backing(size, stride, off), generator=torch.Generator().manual_seed(seed)).to(DEV, dtype)
    return buf.as_strided(size, stride, off)


def assert_same(a, b, what):
    """bitwise equality, NaN patterns included"""
    assert a.shape == b.shape and a.dtype == b.dtype, what
    av, bv = a.detach().contiguous(), b.detach().contiguous()
    iv = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}[a.dtype]
    eq = torch.equal(av.view(iv), bv.view(iv))
    assert eq, (what, (av.float() - bv.float()).abs().max().item())


# ---- module configs ---------------------------------------------------------------------------------------------------

# name -> (module class name, I, H, kwargs, dtype, B, T)
CONFIGS = {
    "gru256": ("GRU", 256, 256, {}, torch.float32, 128, 5),            # streamed, in-place projection at B = 128
    "gru128": ("GRU", 128, 128, {}, torch.float32, 32, 5),
    "bilstm128": ("LSTM", 128, 128, {"bidirectional": True}, torch.float32, 32, 5),
    "lstm_proj": ("LSTM", 128, 256, {"proj_size": 64}, torch.float32, 32, 5),
    "gru272": ("GRU", 64, 272, {}, torch.float32, 16, 5),               # runtime-sized recurrence, FFMA projection
    "lstm464": ("LSTM", 64, 464, {}, torch.float32, 16, 4),
    "tanh_i40": ("RNN", 40, 64, {}, torch.float32, 16, 5),              # FFMA projection, vector loads when aligned
    "tanh_i30": ("RNN", 30, 64, {}, torch.float32, 16, 5),              # I % 4 != 0: scalar loads
    "gru256_f16": ("GRU", 256, 256, {}, torch.float16, 32, 5),          # native 16-bit projection (TMA or copy16)
    "gru256_bf16": ("GRU", 256, 256, {}, torch.bfloat16, 32, 5),
    "gru464_f16": ("GRU", 256, 464, {}, torch.float16, 16, 4),          # 3 * 464 % 128 != 0: widen16 + FFMA
    "lstm464_bf16": ("LSTM", 256, 464, {}, torch.bfloat16, 16, 4),
    "gru2_drop": ("GRU", 128, 128, {"num_layers": 2, "dropout": 0.3}, torch.float32, 32, 5),
}

FP32_LAYOUTS = ["pad8", "off1", "bgap", "bsub", "tgap", "bcast_b", "bcast_t", "b1", "t1"]
H16_LAYOUTS = ["pad8", "off1", "off3", "bgap", "bsub", "tgap", "bcast_b", "bcast_t", "b1", "t1"]


def layouts_of(name):
    return H16_LAYOUTS if CONFIGS[name][4] != torch.float32 else FP32_LAYOUTS


def make_module(name, batch_first=False, seed=0):
    import b200rnn

    cls, I, H, kw, dt, _, _ = CONFIGS[name]
    torch.manual_seed(seed)
    m = getattr(b200rnn, cls)(I, H, batch_first=batch_first, **kw).to(DEV, dt)
    return m.train()


def route_of(name, layout, B):
    """the A-operand route the layer-0 input projection of config `name` is meant to take for x in `layout`"""
    cls, I, H, kw, dt, _, _ = CONFIGS[name]
    G = {"GRU": 3, "LSTM": 4, "RNN": 1}[cls] * H
    tiles = B % 128 == 0 or 128 % B == 0
    if layout == "b1":
        B = 1
    if dt != torch.float32:
        if G % 128:
            return "widen"
        in_place = layout in ("dense", "pad8", "bgap", "bsub", "tgap", "t1") and (tiles or layout == "t1")
        return "tma" if in_place else "copy16"
    if I % 32 or G % 128:   # FFMA GEMM, A read through its row map: float4 loads when base and row strides allow
        _, (st, sb, _), off = x_layout(layout, 2, B, I)
        vec = off % 4 == 0 and st % 4 == 0 and sb % 4 == 0
        return "rows/" + ("vec4" if vec else "scalar")
    # t1: a single step is a dense [B][I] block whatever its time stride
    in_place = layout in ("dense", "pad8", "bgap", "bsub", "tgap", "t1") and (tiles or layout == "t1")
    return "tma" if in_place else "gather"


# ---- module forward + backward: the view against its dense copy --------------------------------------------------------

def run_module(m, x, rng, hx=None, lengths=None, dy_of=None):
    """forward + backward of module `m` on x (a leaf), from dropout state `rng`; returns every output and gradient.
    dy_of(y) -> the output gradient (default: a fixed random tensor); the states get fixed random gradients"""
    from b200rnn.functional import rnn_forward

    m.zero_grad(set_to_none=True)
    m._rng_state.copy_(rng)
    if lengths is None:
        out = m(x, hx)
    else:
        out = rnn_forward(x, m._flat_weights, m._config(), m._rng_state, lengths=lengths, hx=hx)
    y, states = out[0], out[1] if len(out) == 2 else out[1:]
    states = states if isinstance(states, tuple) else (states,)
    g = torch.Generator().manual_seed(7)
    dy = dy_of(y) if dy_of else torch.randn(y.shape, generator=g).to(DEV, y.dtype)
    ds = [torch.randn(s.shape, generator=g).to(DEV, s.dtype) for s in states]
    torch.autograd.backward([y, *states], [dy, *ds])
    res = {"y": y, **{k: s for k, s in zip(("h_n", "c_n"), states)}, "dx": x.grad}
    res.update({"d" + n: p.grad for n, p in m.named_parameters()})
    if hx is not None:
        res.update({k: s.grad for k, s in zip(("dh_0", "dc_0"), hx if isinstance(hx, tuple) else (hx,))})
    return res


def compare(name, layout, batch_first, hx=False, ragged=False):
    m = make_module(name, batch_first)
    _, I, H, kw, dt, B, T = CONFIGS[name]
    size, stride, off = x_layout(layout, T, B, I)
    T, B = size[0], size[1]
    view = backed(size, stride, off, dt, seed=11)
    before = view._base.clone() if view._base is not None else None
    xs = view.transpose(0, 1) if batch_first else view
    x = xs.detach().requires_grad_(True)        # keeps the view's strides and storage offset
    xd = xs.detach().contiguous().requires_grad_(True)
    rng = m._rng_state.clone()
    h0 = None
    if hx:
        D = 2 if kw.get("bidirectional") else 1
        L = kw.get("num_layers", 1)
        g = torch.Generator().manual_seed(5)
        h0 = (0.5 * torch.randn(L * D, B, kw.get("proj_size") or H, generator=g)).to(DEV, dt).requires_grad_(True)
        if CONFIGS[name][0] == "LSTM":
            h0 = (h0, (0.5 * torch.randn(L * D, B, H, generator=g)).to(DEV, dt).requires_grad_(True))
    lengths = None
    if ragged:
        lengths = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(3))
        lengths[0] = T
    hx_d = None if h0 is None else tuple(s.detach().clone().requires_grad_(True) for s in h0) if isinstance(
        h0, tuple) else h0.detach().clone().requires_grad_(True)
    got = run_module(m, x, rng, h0, lengths)
    want = run_module(m, xd, rng, hx_d, lengths)
    assert set(got) == set(want)
    for k in want:
        if want[k] is None:
            assert got[k] is None, k
        else:
            assert_same(got[k], want[k], (name, layout, batch_first, k))
    if before is not None:   # the caller's x is never written (ragged: the padding is zeroed in scratch)
        assert_same(view._base, before, "x written")


@pytest.mark.parametrize("batch_first", [False, True], ids=["tm", "bf"])
@pytest.mark.parametrize("layout", FP32_LAYOUTS)
@pytest.mark.parametrize("name", ["gru256", "bilstm128", "tanh_i40"])
def test_fp32_x_layouts_match_dense_bitwise(name, layout, batch_first):
    compare(name, layout, batch_first)


@pytest.mark.parametrize("layout", ["pad8", "off1", "bgap", "bcast_b", "b1", "t1"])
@pytest.mark.parametrize("name", ["gru128", "lstm_proj", "gru272", "lstm464", "tanh_i30"])
def test_more_configs_x_layouts_match_dense_bitwise(name, layout):
    compare(name, layout, batch_first=True)


@pytest.mark.parametrize("batch_first", [False, True], ids=["tm", "bf"])
@pytest.mark.parametrize("layout", H16_LAYOUTS)
@pytest.mark.parametrize("name", ["gru256_f16", "gru256_bf16", "gru464_f16", "lstm464_bf16"])
def test_16bit_x_layouts_match_dense_bitwise(name, layout, batch_first):
    compare(name, layout, batch_first)


@pytest.mark.parametrize("layout", ["bgap", "bsub"])
@pytest.mark.parametrize("B", [32, 96, 128, 256])
def test_batch_gaps_at_every_box_shape(B, layout):
    """B dividing 128 (box of B rows), 128 and a multiple of it (box of 128), and 96 (the gather copy)"""
    saved = CONFIGS["gru256"]
    CONFIGS["gru256"] = saved[:5] + (B, 4)
    try:
        compare("gru256", layout, batch_first=True)
    finally:
        CONFIGS["gru256"] = saved


@pytest.mark.parametrize("layout", ["off1", "bgap", "bcast_t"])
@pytest.mark.parametrize("case", ["ragged", "hx", "two_layers_dropout"])
def test_ragged_hx_and_dropout_with_strided_x(case, layout):
    if case == "ragged":
        compare("bilstm128", layout, batch_first=True, ragged=True)
    elif case == "hx":
        compare("gru256", layout, batch_first=False, hx=True)
    else:
        compare("gru2_drop", layout, batch_first=True)


@pytest.mark.parametrize("layout", ["off1", "bgap", "bcast_b"])
def test_autocast_module_with_strided_x(layout):
    with torch.autocast("cuda", dtype=torch.float16):
        compare("gru256", layout, batch_first=True)


# ---- dy through autograd ------------------------------------------------------------------------------------------------

def dy_layout(name, T, B, C, batch_first):
    """(size, stride, offset) of an output gradient in the module's layout ([B,T,C] batch-first, else [T,B,C])"""
    sz = (B, T, C) if batch_first else (T, B, C)
    if name == "stride_t0":
        return sz, ((C, 0, 1) if batch_first else (0, C, 1)), 0
    if name == "both0":
        return sz, (0, 0, 1), 0
    if name == "stride_b0":
        return sz, ((0, C, 1) if batch_first else (C, 0, 1)), 0
    if name == "gapped":
        return sz, ((2 * T * C, C, 1) if batch_first else (B * 2 * C, 2 * C, 1)), 0
    if name == "misaligned":
        return sz, ((T * (C + 1), C + 1, 1) if batch_first else (B * (C + 1), C + 1, 1)), 1
    raise KeyError(name)


@pytest.mark.parametrize("dy", ["stride_t0", "both0", "stride_b0", "gapped", "misaligned"])
@pytest.mark.parametrize("batch_first", [False, True], ids=["tm", "bf"])
@pytest.mark.parametrize("name", ["gru256", "bilstm128", "gru272", "gru256_f16"])
def test_dy_layouts_match_dense_bitwise(name, batch_first, dy):
    m = make_module(name, batch_first)
    _, I, H, kw, dt, B, T = CONFIGS[name]
    C = (2 if kw.get("bidirectional") else 1) * (kw.get("proj_size") or H)
    xv = backed((T, B, I), (B * I, I, 1), 0, dt, seed=11)
    xs = xv.transpose(0, 1) if batch_first else xv
    size, stride, off = dy_layout(dy, T, B, C, batch_first)
    g = backed(size, stride, off, dt, seed=13)
    rng = m._rng_state.clone()
    x1, x2 = xs.detach().clone().requires_grad_(True), xs.detach().clone().requires_grad_(True)
    got = run_module(m, x1, rng, dy_of=lambda y: g)
    want = run_module(m, x2, rng, dy_of=lambda y: g.contiguous())
    for k in want:
        assert_same(got[k], want[k], (name, dy, k))


@pytest.mark.parametrize("reduce", ["time", "time_and_batch"])
def test_dy_from_autograd_sums(reduce):
    """y.sum(time) / y.sum((0, 1)) give the backward a dy with stride_t = 0 (and stride_b = 0)"""
    m = make_module("gru256", batch_first=False)
    _, I, H, _, _, B, T = CONFIGS["gru256"]
    x = backed((T, B, I), (B * I, I, 1), 0, torch.float32, seed=11).detach()
    w = torch.randn(B, H, generator=torch.Generator().manual_seed(2)).to(DEV)
    outs = []
    for expand in (False, True):
        m.zero_grad(set_to_none=True)
        xx = x.clone().requires_grad_(True)
        y = m(xx)[0]
        if reduce == "time":
            loss = (y.sum(0) * w).sum() if not expand else (y * w.expand(T, B, H).contiguous()).sum()
        else:
            loss = y.sum((0, 1)).mul(w[0]).sum() if not expand else (y * w[0].expand(T, B, H).contiguous()).sum()
        loss.backward()
        outs.append({"dx": xx.grad, **{n: p.grad for n, p in m.named_parameters()}})
    for k in outs[1]:
        assert_same(outs[0][k], outs[1][k], (reduce, k))


# ---- forward_ln_sum, the frozen weight cache, rnn_ln_pool_sum ------------------------------------------------------------

def _ln_case(layout, batch_first, grad, frozen=False):
    import b200rnn

    torch.manual_seed(0)
    gru = b200rnn.GRU(256, 256, batch_first=batch_first).to(DEV)
    ln = torch.nn.LayerNorm(256).to(DEV)
    with torch.no_grad():
        ln.weight.uniform_(0.5, 1.5)
        ln.bias.uniform_(-0.5, 0.5)
    if frozen:
        for p in gru.parameters():
            p.requires_grad_(False)
    T, B = 6, 32
    size, stride, off = x_layout(layout, T, B, 256)
    view = backed(size, stride, off, torch.float32, seed=21)
    xs = view.transpose(0, 1) if batch_first else view
    res = []
    for x in (xs.detach(), xs.detach().contiguous()):
        gru.zero_grad(set_to_none=True)
        ln.zero_grad(set_to_none=True)
        x = x.requires_grad_(grad)
        with torch.set_grad_enabled(grad):
            out = gru.forward_ln_sum(x, ln)
            r = {"out": out}
            if grad:
                out.mul(torch.linspace(-1, 1, out.numel(), device=DEV).view_as(out)).sum().backward()
                r["dx"] = x.grad
                r.update({n: p.grad for n, p in [*gru.named_parameters(), *ln.named_parameters()]})
        res.append(r)
    for k in res[1]:
        assert_same(res[0][k], res[1][k], (layout, grad, k))


@pytest.mark.parametrize("grad", [False, True], ids=["nograd", "grad"])
@pytest.mark.parametrize("batch_first", [False, True], ids=["tm", "bf"])
@pytest.mark.parametrize("layout", ["off1", "pad8", "bgap", "t1", "bcast_b"])
def test_forward_ln_sum_on_strided_x_matches_dense_bitwise(layout, batch_first, grad):
    """the LayerNorm fold reads x in place only when it is 16-byte aligned row by row; any other x runs on a dense
    copy (b200rnn.functional._ln_operands) instead of failing in the library"""
    _ln_case(layout, batch_first, grad)


@pytest.mark.parametrize("layout", ["off1", "bgap"])
def test_frozen_weight_cache_no_grad_on_strided_x(layout):
    _ln_case(layout, True, False, frozen=True)


def test_rnn_ln_pool_sum_offset_x():
    """the functional entry directly, on x at an offset of one float"""
    import b200rnn
    from b200rnn.functional import rnn_ln_pool_sum

    torch.manual_seed(0)
    gru = b200rnn.GRU(256, 128, bidirectional=True).to(DEV)
    ln_w = torch.rand(256, device=DEV) + 0.5
    ln_b = torch.rand(256, device=DEV) - 0.5
    view = backed(*x_layout("off1", 5, 32, 256), torch.float32, seed=3)
    res = []
    for x in (view.detach(), view.detach().contiguous()):
        gru.zero_grad(set_to_none=True)
        x = x.requires_grad_(True)
        w, b = ln_w.clone().requires_grad_(True), ln_b.clone().requires_grad_(True)
        out = rnn_ln_pool_sum(x, gru._flat_weights, gru._config(), gru._rng_state, None, w, b, 1e-5)
        out.pow(2).sum().backward()
        res.append({"out": out, "dx": x.grad, "dw": w.grad, "db": b.grad,
                    **{n: p.grad for n, p in gru.named_parameters()}})
    for k in res[1]:
        assert_same(res[0][k], res[1][k], k)


# ---- the C ABI: y and dx into caller buffers --------------------------------------------------------------------------

def sentinel_view(size, stride, off, dtype):
    """a view over a buffer filled with the sentinel bit pattern, and a mask of the view's elements in that buffer"""
    n = backing(size, stride, off)
    if dtype == torch.float32:
        buf = torch.full((n,), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
    else:
        buf = torch.full((n,), SENTINEL16, dtype=torch.int16, device=DEV).view(dtype)
    mask = torch.zeros(n, dtype=torch.bool, device=DEV)
    mask.as_strided(size, stride, off).fill_(True)
    return buf, buf.as_strided(size, stride, off), mask


def assert_untouched(buf, mask, what):
    iv, want = (torch.int32, SENTINEL) if buf.dtype == torch.float32 else (torch.int16, SENTINEL16)
    outside = buf.view(iv)[~mask]
    assert bool((outside == want).all()), (what, int((outside != want).sum()))


def out_layout(kind, T, B, C):
    """time-major [T,B,C] output buffer: dense, gapped (time and row gaps), a time gap only, or one element off"""
    if kind == "dense":
        return (T, B, C), (B * C, C, 1), 0
    if kind == "gapped":
        return (T, B, C), (2 * B * (C + 8), C + 8, 1), 0
    if kind == "tgap":
        return (T, B, C), (2 * B * C, C, 1), 0
    return (T, B, C), (B * (C + 1), C + 1, 1), 1


def abi_fwd_bwd(m, x, y_kind, dx_kind, dy, fused=False):
    """b200rnn_forward_hx (or _fused) into a y of `y_kind` and b200rnn_backward_hx (or _fused) into a dx of `dx_kind`,
    both pre-filled with the sentinel; x, dy time-major views. Returns y, dx, h_n, weight gradients and the buffers"""
    from b200rnn import _lib
    from b200rnn.functional import _make_desc, _stream_ptr

    lib = _lib.load()
    cfg = m._config()
    T, B, I = x.shape
    C = cfg.num_dirs * cfg.out_size
    desc = _make_desc(cfg, B, T, True)
    rbytes, sbytes = _lib.workspace_bytes(desc)
    reserve = torch.empty(rbytes, dtype=torch.uint8, device=DEV)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=DEV)
    ybuf, y, ymask = sentinel_view(*out_layout(y_kind, T, B, C), x.dtype)
    L, D = cfg.num_layers, cfg.num_dirs
    h_n = torch.empty(L * D, B, cfg.out_size, dtype=x.dtype, device=DEV)
    c_n = torch.empty(L * D, B, cfg.hidden_size, dtype=x.dtype, device=DEV) if cfg.mode == _lib.LSTM else None
    params = _lib.ptr_array([w.data_ptr() for w in m._flat_weights])
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    st = _stream_ptr(DEV)
    if fused:
        rc = lib.b200rnn_forward_fused(ctypes.byref(desc), x.data_ptr(), x.stride(0), x.stride(1), params,
                                       y.data_ptr(), y.stride(0), y.stride(1), h_n.data_ptr(), ptr(c_n),
                                       reserve.data_ptr(), scratch.data_ptr(), 0, 0, m._rng_state.data_ptr(),
                                       None, None, 1e-5, None, None, None, None, st)
    else:
        rc = lib.b200rnn_forward_hx(ctypes.byref(desc), x.data_ptr(), x.stride(0), x.stride(1), params,
                                    y.data_ptr(), y.stride(0), y.stride(1), None, None, h_n.data_ptr(), ptr(c_n),
                                    reserve.data_ptr(), scratch.data_ptr(), 0, 0, m._rng_state.data_ptr(), None, st)
    _lib.check(rc, "forward")
    dxbuf, dx, dxmask = sentinel_view(*out_layout(dx_kind, T, B, I), x.dtype)
    grads = [torch.empty_like(w) for w in m._flat_weights]
    dparams = _lib.ptr_array([g.data_ptr() for g in grads])
    if fused:
        rc = lib.b200rnn_backward_fused(ctypes.byref(desc), x.data_ptr(), x.stride(0), x.stride(1), params,
                                        y.data_ptr(), y.stride(0), y.stride(1), dy.data_ptr(), dy.stride(0),
                                        dy.stride(1), None, 0.0, None, None, reserve.data_ptr(), scratch.data_ptr(),
                                        dx.data_ptr(), dx.stride(0), dx.stride(1), dparams, None, None, 1e-5, None,
                                        None, st)
    else:
        rc = lib.b200rnn_backward_hx(ctypes.byref(desc), x.data_ptr(), x.stride(0), x.stride(1), params,
                                     y.data_ptr(), y.stride(0), y.stride(1), dy.data_ptr(), dy.stride(0),
                                     dy.stride(1), None, None, None, None, None, None, reserve.data_ptr(),
                                     scratch.data_ptr(), dx.data_ptr(), dx.stride(0), dx.stride(1), dparams, None, st)
    _lib.check(rc, "backward")
    torch.cuda.synchronize()
    return {"y": y, "dx": dx, "h_n": h_n, **{"d%d" % i: g for i, g in enumerate(grads)}}, (ybuf, ymask), (dxbuf, dxmask)


ABI_CONFIGS = ["gru256", "tanh_i40", "gru272", "gru256_f16"]


# the _fused pair takes fp32 GRU / LSTM at hidden sizes 128 and 256 only
# (config, y / dx layout, _fused pair, dy layout): a gapped dy beside gapped outputs, a misaligned one beside outputs
# one element off, and the broadcast dy of the catalogue straight into the C ABI
ABI_CASES = [(n, o, f, "misaligned" if o == "off1" else "gapped") for n in ABI_CONFIGS
             for o in ("gapped", "tgap", "off1") for f in (False, True) if not f or n == "gru256"]
ABI_CASES += [(n, "gapped", False, d) for n in ABI_CONFIGS for d in ("stride_t0", "both0", "stride_b0")]


@pytest.mark.parametrize("name,out,fused,dy_kind", ABI_CASES)
def test_abi_outputs_into_strided_buffers(name, out, fused, dy_kind):
    m = make_module(name).eval()
    _, I, H, kw, dt, B, T = CONFIGS[name]
    C = (2 if kw.get("bidirectional") else 1) * H
    x = backed(*x_layout("off1" if out == "off1" else "bgap", T, B, I), dt, seed=31)
    dy = backed(*dy_layout(dy_kind, T, B, C, False), dt, seed=32)
    x0, dy0 = x._base.clone(), dy._base.clone()
    rng = m._rng_state.clone()
    got, (ybuf, ymask), (dxbuf, dxmask) = abi_fwd_bwd(m, x, out, out, dy, fused)
    m._rng_state.copy_(rng)
    want, _, _ = abi_fwd_bwd(m, x.contiguous(), "dense", "dense", dy.contiguous(), fused)
    assert_untouched(ybuf, ymask, "y")
    assert_untouched(dxbuf, dxmask, "dx")
    assert_same(x._base, x0, "x written")
    assert_same(dy._base, dy0, "dy written")
    # a dx one element off cannot take the tensor-core dgrad epilogue (16-byte aligned rows): FFMA, same operands
    tc_dgrad = dt == torch.float32 and I % 128 == 0
    for k in want:
        if k == "dx" and out == "off1" and tc_dgrad:
            continue
        assert_same(got[k], want[k], (name, out, k))
    if out == "off1" and tc_dgrad:   # the FFMA dgrad against float64, with the bound of test_gpu_numerics_f64.py
        ref = getattr(torch.nn, CONFIGS[name][0])(I, H, **kw)
        ref.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()})
        xc, wy = x.detach().float().cpu().contiguous(), dy.detach().float().cpu().contiguous()
        hx = [torch.zeros(1, B, H)]
        ws = [torch.zeros(1, B, H)]
        r64 = _run_torch(ref, xc, None, hx, wy, ws, torch.float64)
        r32 = _run_torch(ref, xc, None, hx, wy, ws, torch.float32)
        e_mine = _norm_err(got["dx"].double().cpu().numpy(), r64["dx"])
        e_tc = _norm_err(want["dx"].double().cpu().numpy(), r64["dx"])
        e_t = _norm_err(r32["dx"], r64["dx"])
        assert e_mine <= 4 * e_t + 1e-6 and e_tc <= 4 * e_t + 1e-6, (e_mine, e_tc, e_t)


# ---- every layout on its intended route -------------------------------------------------------------------------------

_ROUTE_CHILD = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}, {tests!r}]
import torch
import test_gpu_strided_io as t
for name, layout, B in {cases!r}:
    saved = t.CONFIGS[name]
    t.CONFIGS[name] = saved[:5] + (B, saved[6])
    m = t.make_module(name).eval()
    _, I, H, kw, dt, _, T = t.CONFIGS[name]
    x = t.backed(*t.x_layout(layout, T, B, I), dt, seed=1)
    with torch.no_grad():
        m(x)
    torch.cuda.synchronize()
    t.CONFIGS[name] = saved
    print("[b200rnn] ran", name, layout, B, file=sys.stderr, flush=True)
gru = t.make_module("gru256").eval()
ln = torch.nn.LayerNorm(256).to("cuda:0")
with torch.no_grad():
    gru.forward_ln_sum(t.backed(*t.x_layout("pad8", 5, 32, 256), torch.float32, seed=1), ln)
torch.cuda.synchronize()
print("[b200rnn] ran gru256 ln 32", file=sys.stderr, flush=True)
"""


def route_cases():
    cases = []
    for name in CONFIGS:
        if name == "gru2_drop":
            continue
        for layout in ["dense"] + layouts_of(name):
            cases.append((name, layout, CONFIGS[name][5]))
    for B in (32, 96, 128, 256):
        for layout in ("bgap", "bsub", "pad8"):
            cases.append(("gru256", layout, B))
    return cases


def test_routes():
    cases = route_cases()
    env = dict(os.environ, B200RNN_DEBUG="1")
    code = _ROUTE_CHILD.format(root=ROOT, pkg=PKG, tests=os.path.dirname(os.path.abspath(__file__)), cases=cases)
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr[-4000:]
    seen, first = {}, None
    for ln in proc.stderr.splitlines():
        if ln.startswith(("[b200rnn] forward x-projection:", "[b200rnn] ffma x-projection:")) and first is None:
            kv = dict(w.split("=", 1) for w in ln.split()[3:] if "=" in w)
            first = kv["a"] + ("/" + kv["loads"] if kv["a"] == "rows" else "")
        elif ln.startswith("[b200rnn] ran "):
            _, _, name, layout, B = ln.split()
            seen[(name, layout, int(B))] = first
            first = None
    want = {(n, lay, B): route_of(n, lay, B) for n, lay, B in cases}
    want[("gru256", "ln", 32)] = "ln"
    bad = {k: (seen.get(k), v) for k, v in want.items() if seen.get(k) != v}
    assert not bad, bad
    # the catalogue reaches every route word of the projection's A operand
    assert {v.split("/")[0] for v in seen.values()} == {"tma", "gather", "ln", "copy16", "widen", "rows"}
    assert {v for v in seen.values() if v.startswith("rows/")} == {"rows/vec4", "rows/scalar"}
