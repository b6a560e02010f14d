"""Autograd bridge between PyTorch tensors and the C-ABI library.

``rnn_forward`` is what ``b200rnn.GRU.forward`` / ``b200rnn.LSTM.forward`` call in place of ``_VF.gru`` /
``_VF.lstm`` (torch/nn/modules/rnn.py:1449 / :1169). PyTorch is only plumbing here: it owns the device
memory (``torch.empty`` -> caching allocator, CUDA-graph friendly) and the current stream; all arithmetic
happens in ``lib/libb200rnn.so``. CPU tensors are rejected — there is no fallback path.
"""
from __future__ import annotations

import ctypes
import dataclasses
from dataclasses import dataclass
from typing import Optional, Sequence

import torch
import torch.autograd.forward_ad as fwAD

from . import _lib

# rnn_forward's `save` when forward-mode AD may ask for a tangent: the forward keeps its reserve whatever autograd needs
SAVE_FOR_TANGENT = 2


@dataclass
class RNNConfig:
    mode: int            # _lib.GRU / _lib.LSTM
    input_size: int
    hidden_size: int
    num_layers: int
    num_dirs: int
    dropout: float
    training: bool
    batch_first: bool
    tf32: bool = False   # single-pass TF32 tensor-core GEMMs / tc8 recurrence (tf32_enabled()), else 3xTF32
    proj_size: int = 0   # LSTM with projections: width P of h_t (0 = none)
    dtype: torch.dtype = torch.float32   # of x, the parameters, the states and every output (16-bit: FLAG_F16 / _BF16)
    # fp32 master parameters of a 16-bit call (torch.autocast, FLAG_F32_PARAMS): the parameters and their gradients
    # are float32, everything else is ``dtype``; computes what the 16-bit module computes on the rounded parameters
    master_f32: bool = False
    # M > 1: one call runs M models (torch.func.vmap, b200rnn.func): x [M,T,B,I] (or [M,B,T,I]), every parameter
    # [M, ...] (model stride 0 = shared), h_0 / c_0 and every output and gradient dense [M, ...]
    models: int = 1
    # with models > 1, the model stride of rng_state: 2 = one row per model, 0 = one state and one mask for every
    # model, -1 = one state drawn by the models as consecutive calls would draw it
    rng_stride: int = 0

    @property
    def out_size(self) -> int:
        """width of h_t and of the output per direction: proj_size, or hidden_size without a projection"""
        return self.proj_size if self.proj_size > 0 else self.hidden_size


@torch.compiler.assume_constant_result   # dynamo cannot read the setting: a compiled graph keeps the value it traced
def tf32_enabled() -> bool:
    """Whether torch's fp32 matmul precision asks for TF32: ``torch.backends.cuda.matmul.fp32_precision``, or, while
    that is ``"none"``, the global ``torch.backends.fp32_precision``. ``torch.set_float32_matmul_precision("high")``
    sets the former to ``"tf32"``, ``"highest"`` to ``"ieee"``; the default ``"none"`` / ``"ieee"`` keeps 3xTF32.
    (``torch.get_float32_matmul_precision()`` is not used: it raises once both the legacy and the new API have been
    used in a process.) The cuDNN RNN knob, which defaults to TF32, is deliberately not followed."""
    mode = torch.backends.cuda.matmul.fp32_precision
    if mode == "none":
        mode = torch.backends.fp32_precision
    return mode == "tf32"


def _require_cuda_f32(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise _lib.NoCPUPathError(
            f"b200rnn: {name} is on {t.device}; this library runs on CUDA (sm_90a) only and has no CPU path"
        )
    if t.dtype != torch.float32:
        raise _lib.B200RNNError(f"b200rnn: {name} must be float32 (got {t.dtype})")


def _require_cuda_dtype(t: torch.Tensor, name: str, dtype: torch.dtype) -> None:
    """float32 calls: as _require_cuda_f32. 16-bit calls: every tensor has the call's dtype (the parameters' dtype, or
    float32 for the parameters of a master-weight call)"""
    if dtype == torch.float32:
        _require_cuda_f32(t, name)
        return
    if not t.is_cuda:
        raise _lib.NoCPUPathError(
            f"b200rnn: {name} is on {t.device}; this library runs on CUDA (sm_90a) only and has no CPU path"
        )
    if t.dtype != dtype:
        raise _lib.B200RNNError(f"b200rnn: {name} must be {dtype} like the first weight (got {t.dtype})")


def _tm_view(x: torch.Tensor) -> torch.Tensor:
    """Return a logical [T,B,F] tensor whose feature stride is 1 (copy only if it is not)."""
    if x.stride(2) != 1 and x.size(2) != 1:
        x = x.contiguous()
    return x


def _ln_operand_ok(x_tm: torch.Tensor, ln_w: Optional[torch.Tensor], ln_b: Optional[torch.Tensor]) -> bool:
    """Whether the fused LayerNorm prologue and its backward can read ``x_tm`` [T,B,I] as it lies: a 16-byte aligned
    base, time and batch strides that are multiples of 4 floats, and 16-byte aligned gamma and beta. The C ABI returns
    ``B200RNN_ERR_UNSUPPORTED`` for any other x; the Python entries run on a dense copy instead."""
    def aligned(t):
        return t is None or t.data_ptr() % 16 == 0
    return aligned(x_tm) and x_tm.stride(0) % 4 == 0 and x_tm.stride(1) % 4 == 0 and aligned(ln_w) and aligned(ln_b)


def _ln_operands(x_tm: torch.Tensor, ln_w: Optional[torch.Tensor], ln_b: Optional[torch.Tensor]):
    """``(x_tm, ln_w, ln_b)`` as the fused LayerNorm reads them: each tensor :func:`_ln_operand_ok` rejects is replaced
    by a fresh (aligned; for x, dense time-major) copy, the others are passed as they are. The copies are
    differentiable: autograd carries dx, dgamma and dbeta back to the caller's tensors."""
    if ln_w is None or _ln_operand_ok(x_tm, ln_w, ln_b):
        return x_tm, ln_w, ln_b
    fresh = lambda t: t if t is None or t.data_ptr() % 16 == 0 else t.clone()  # noqa: E731
    if not _ln_operand_ok(x_tm, None, None):
        x_tm = x_tm.clone(memory_format=torch.contiguous_format)
    return x_tm, fresh(ln_w), fresh(ln_b)


def _make_desc(cfg: RNNConfig, B: int, T: int, save: bool, accumulate: bool = False,
               fused_ln: bool = False, model_strides: Optional[Sequence[int]] = None) -> _lib.Desc:
    """``model_strides`` (``cfg.models > 1``): of x, rng_state and each parameter, in elements (zeros when None: the
    workspace sizes do not depend on them)"""
    flags = 0
    if save:
        flags |= _lib.FLAG_SAVE_FOR_BACKWARD
    if accumulate:
        flags |= _lib.FLAG_ACCUMULATE_GRADS
    if fused_ln:
        flags |= _lib.FLAG_FUSED_LN
    if cfg.tf32:
        flags |= _lib.FLAG_TF32
    if cfg.proj_size:
        flags |= _lib.FLAG_PROJ
    flags |= _lib.H16_DTYPES.get(str(cfg.dtype), 0)
    if cfg.master_f32:
        flags |= _lib.FLAG_F32_PARAMS
    desc = _lib.Desc(cfg.mode, B, T, cfg.input_size, cfg.hidden_size, cfg.num_layers, cfg.num_dirs,
                     1 if cfg.training else 0, float(cfg.dropout), flags, cfg.proj_size)
    if cfg.models > 1:
        n = 2 + 4 * cfg.num_layers * cfg.num_dirs
        strides = (ctypes.c_int64 * n)(*(model_strides if model_strides is not None else [0] * n))
        desc.flags |= _lib.FLAG_MODELS
        desc.models = cfg.models
        desc.model_strides = ctypes.cast(strides, ctypes.POINTER(ctypes.c_int64))
        desc.keepalive = strides   # the library reads the array during the call
    return desc


def _model_strides(cfg: RNNConfig, x_tm: torch.Tensor, weights: Sequence[torch.Tensor]) -> Optional[list]:
    """the model strides of a ``cfg.models > 1`` call: x, rng_state, each parameter (None for one model)"""
    if cfg.models == 1:
        return None
    return [x_tm.stride(0), cfg.rng_stride, *(w.stride(0) for w in weights)]


def _stream_ptr(device=None) -> int:
    """Raw handle of the current stream OF ``device`` (not of the process-wide current device)."""
    return torch.cuda.current_stream(device).cuda_stream


def _on(device):
    """Make ``device`` current around a library call: the C side queries / configures the CURRENT device
    (``cudaFuncSetAttribute``, occupancy, SM count), and stock nn.GRU / nn.LSTM work on whatever device their tensors
    live on, so the drop-in has to as well (module on cuda:1 while cuda:0 is the process default)."""
    return torch.cuda.device(device)


def _weight_grad_targets(weights, needed, sink, dev, separate: bool = False):
    """Where a backward writes the weight gradients, as ``(dptrs, grads_out, accumulate)``: straight into the views
    ``sink(weights)`` returns (a flat all-reduce bucket; the kernels accumulate into them, ``grads_out`` is all None),
    or into one fresh flat buffer (in the weights' dtype) whose views are returned to autograd. ``needed[i]``: whether
    ``weights[i]`` wants a gradient (a NULL target otherwise). Each fresh view starts on a 256-byte boundary.
    ``separate``: one fresh tensor per gradient instead (the custom ops, whose outputs may not alias each other)."""
    if sink is not None:
        targets = sink(weights)  # list of tensors (same shapes) or None entries
        dptrs = [t.data_ptr() if (t is not None and n) else None for t, n in zip(targets, needed)]
        return dptrs, [None] * len(weights), True
    if separate:
        grads_out = _weight_grad_buffers(weights, needed)
        return [g.data_ptr() if g is not None else None for g in grads_out], grads_out, False
    align = 256 // weights[0].element_size()
    sizes = [(w.numel() + align - 1) // align * align if n else 0 for w, n in zip(weights, needed)]
    flat = torch.empty(sum(sizes), dtype=weights[0].dtype, device=dev)
    grads_out, off = [], 0
    for w, n, size in zip(weights, needed, sizes):
        grads_out.append(flat[off:off + w.numel()].view_as(w) if n else None)
        off += size
    return [g.data_ptr() if g is not None else None for g in grads_out], grads_out, False


def _weight_grad_buffers(weights, needed):
    """one fresh dense gradient tensor per weight that wants one (None otherwise)"""
    return [torch.empty(w.shape, dtype=w.dtype, device=w.device) if n else None for w, n in zip(weights, needed)]


def _forward_buffers(x_tm: torch.Tensor, cfg: RNNConfig, save: bool, with_scratch: bool = True,
                     model_strides: Optional[Sequence[int]] = None):
    """Descriptor and the buffers of one sequence forward, as ``(desc, reserve, scratch, y, (ys_t, ys_b), h_n, c_n)``:
    ``y`` batch-first or time-major as ``cfg`` says, ``c_n`` None but for the LSTM, the reserve empty without ``save``.
    Host arithmetic only (``b200rnn_workspace_bytes``), so the custom ops' fake implementations call it too, without
    the scratch. With ``cfg.models`` = M > 1 every buffer has a leading [M] dimension (the reserve: M one-model blocks)."""
    T, B = x_tm.shape[-3], x_tm.shape[-2]
    H, L, D, HO = cfg.hidden_size, cfg.num_layers, cfg.num_dirs, cfg.out_size
    dev = x_tm.device
    M = cfg.models
    lead = (M,) if M > 1 else ()
    desc = _make_desc(cfg, B, T, save, model_strides=model_strides)
    rbytes, sbytes = _lib.workspace_bytes(desc)
    reserve = torch.empty(*lead, rbytes // M if save else 0, dtype=torch.uint8, device=dev)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev) if with_scratch else None
    dt = cfg.dtype
    if cfg.batch_first:
        y = torch.empty(*lead, B, T, D * HO, dtype=dt, device=dev)
        ys = (D * HO, T * D * HO)
    else:
        y = torch.empty(*lead, T, B, D * HO, dtype=dt, device=dev)
        ys = (B * D * HO, D * HO)
    h_n = torch.empty(*lead, L * D, B, HO, dtype=dt, device=dev)
    c_n = torch.empty(*lead, L * D, B, H, dtype=dt, device=dev) if cfg.mode == _lib.LSTM else None
    return desc, reserve, scratch, y, ys, h_n, c_n


def _rnn_forward_impl(x_tm: torch.Tensor, cfg: RNNConfig, rng_state: Optional[torch.Tensor],
                      lengths: Optional[torch.Tensor], save: bool, h_0: Optional[torch.Tensor],
                      c_0: Optional[torch.Tensor], weights: Sequence[torch.Tensor]):
    """The sequence forward (one ``b200rnn_forward_hx`` call) shared by :class:`_RNNFunction` and the
    ``b200rnn::rnn_forward`` op: returns ``(y, h_n, c_n, reserve)``, ``c_n`` None but for the LSTM."""
    lib = _lib.load()
    T, B = x_tm.shape[-3], x_tm.shape[-2]
    dev = x_tm.device
    desc, reserve, scratch, y, (ys_t, ys_b), h_n, c_n = _forward_buffers(x_tm, cfg, save,
                                                                         model_strides=_model_strides(cfg, x_tm, weights))
    params = _lib.ptr_array([w.data_ptr() for w in weights])
    rng_ptr = rng_state.data_ptr() if rng_state is not None else None
    len_ptr = lengths.data_ptr() if lengths is not None else None
    c_n_ptr = c_n.data_ptr() if c_n is not None else None
    if B > 0 and T > 0:
        # the module forward, with or without hx: the model-shell entry b200rnn_forward_fused is for
        # rnn_forward_fused / rnn_ln_pool_sum (its no-grad GRU-256 recurrence runs on fp16 pairs)
        with _on(dev):
            rc = lib.b200rnn_forward_hx(
                ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(-3), x_tm.stride(-2), params,
                y.data_ptr(), ys_t, ys_b, h_0.data_ptr() if h_0 is not None else None,
                c_0.data_ptr() if c_0 is not None else None,
                h_n.data_ptr(), c_n_ptr, reserve.data_ptr() if save else None, scratch.data_ptr(),
                0, 0, rng_ptr, len_ptr, _stream_ptr(dev))
        _lib.check(rc, "b200rnn_forward")
    else:   # no step: the final state is the initial one
        h_n.copy_(h_0) if h_0 is not None else h_n.zero_()
        if c_n is not None:
            c_n.copy_(c_0) if c_0 is not None else c_n.zero_()
    return y, h_n, c_n, reserve


def _dx_buffer(x_tm: torch.Tensor) -> torch.Tensor:
    """the input gradient: laid out like ``x_tm`` when its feature stride is 1, else dense time-major; several models
    ([M,T,B,I]): dense"""
    if x_tm.dim() == 4:
        return torch.empty(x_tm.shape, dtype=x_tm.dtype, device=x_tm.device)
    dx = torch.empty_like(x_tm)
    if dx.stride(2) != 1 and dx.size(2) != 1:
        dx = torch.empty(x_tm.shape, dtype=x_tm.dtype, device=x_tm.device)
    return dx


def _rnn_backward_impl(cfg: RNNConfig, x_tm, y, reserve, h_0, c_0, weights, dy, dh_n, dc_n, lengths,
                       need_dx: bool, need_dh_0: bool, need_dc_0: bool, need_w, grad_sink, separate: bool = False):
    """BPTT (``b200rnn_backward`` / ``_hx``) shared by :class:`_RNNFunction` and the ``b200rnn::rnn_backward`` op:
    returns ``(dx, dh_0, dc_0, weight grads)``, None for every gradient that is not wanted (a NULL pointer to the
    library). ``grad_sink`` / ``separate``: see :func:`_weight_grad_targets`."""
    lib = _lib.load()
    T, B = x_tm.shape[-3], x_tm.shape[-2]
    dev = x_tm.device
    if cfg.batch_first:
        ys_t, ys_b = cfg.num_dirs * cfg.out_size, T * cfg.num_dirs * cfg.out_size
    else:
        ys_t, ys_b = B * cfg.num_dirs * cfg.out_size, cfg.num_dirs * cfg.out_size
    # gradients w.r.t. the initial state only when autograd asks: dh_0 costs the last step's contraction
    dh_0 = torch.empty_like(h_0) if h_0 is not None and need_dh_0 else None
    dc_0 = torch.empty_like(c_0) if c_0 is not None and need_dc_0 else None

    if dy is None:
        dy = torch.zeros_like(y)
    if (dy.stride(-1) != 1 and dy.size(-1) != 1) or cfg.models > 1:   # several models: dense per model
        dy = dy.contiguous()
    if cfg.batch_first:
        dys_t, dys_b = dy.stride(-2), dy.stride(-3)
    else:
        dys_t, dys_b = dy.stride(-3), dy.stride(-2)
    if dh_n is not None:
        dh_n = dh_n.contiguous()
    if dc_n is not None:
        dc_n = dc_n.contiguous()

    dx = _dx_buffer(x_tm) if need_dx else None

    dptrs, grads_out, accumulate = _weight_grad_targets(weights, need_w, grad_sink, dev, separate)
    desc = _make_desc(cfg, B, T, True, accumulate, model_strides=_model_strides(cfg, x_tm, weights))
    _, sbytes = _lib.workspace_bytes(desc)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
    params = _lib.ptr_array([w.data_ptr() for w in weights])
    dparams = _lib.ptr_array(dptrs)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    if B > 0 and T > 0:
        with _on(dev):
            head = (ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(-3), x_tm.stride(-2), params,
                    y.data_ptr(), ys_t, ys_b, dy.data_ptr(), dys_t, dys_b, ptr(dh_n), ptr(dc_n))
            tail = (reserve.data_ptr(), scratch.data_ptr(), ptr(dx),
                    dx.stride(-3) if dx is not None else 0, dx.stride(-2) if dx is not None else 0,
                    dparams, ptr(lengths), _stream_ptr(dev))
            if h_0 is None and not cfg.proj_size:
                rc = lib.b200rnn_backward(*head, *tail)
            else:
                rc = lib.b200rnn_backward_hx(*head, ptr(h_0), ptr(c_0), ptr(dh_0), ptr(dc_0), *tail)
        _lib.check(rc, "b200rnn_backward")
    else:   # no step: parameters get nothing, the state gradients pass through
        for g in grads_out:
            if g is not None:
                g.zero_()
        for d0, dn in ((dh_0, dh_n), (dc_0, dc_n)):
            if d0 is not None:
                d0.copy_(dn) if dn is not None else d0.zero_()
    return dx, dh_0, dc_0, grads_out


def _rnn_tangent_impl(cfg: RNNConfig, x_tm, y, reserve, h_0, c_0, weights, x_dot, h0_dot, c0_dot, w_dots,
                      directions: int = 1):
    """Forward-mode AD of a saving forward (one ``b200rnn_forward_tangent`` call): ``(y', h_n', c_n')`` from the
    tangents of x (time-major), h_0, c_0 and each weight, each None = 0. ``y'`` is laid out like ``y``, ``c_n'`` None but
    for the LSTM. ``directions`` = M > 1: every tangent (and output) carries a leading [M] dimension of tangent
    directions over the one primal, which the library runs in one recurrence launch per layer."""
    lib = _lib.load()
    T, B = x_tm.shape[0], x_tm.shape[1]
    H, L, D = cfg.hidden_size, cfg.num_layers, cfg.num_dirs
    dev = x_tm.device
    M = directions
    lead = (M,) if M > 1 else ()
    desc = _make_desc(dataclasses.replace(cfg, models=M), B, T, True)
    sbytes = _lib.tangent_workspace_bytes(desc)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
    y_dot = torch.empty(*lead, *y.shape, dtype=torch.float32, device=dev)
    if cfg.batch_first:
        ys, yds = (D * H, T * D * H), (D * H, T * D * H)
    else:
        ys, yds = (B * D * H, D * H), (B * D * H, D * H)
    h_n_dot = torch.empty(*lead, L * D, B, H, dtype=torch.float32, device=dev)
    c_n_dot = torch.empty(*lead, L * D, B, H, dtype=torch.float32, device=dev) if cfg.mode == _lib.LSTM else None
    dense = lambda t: t.contiguous() if t is not None else None  # noqa: E731
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    x_dot, h0_dot, c0_dot = dense(x_dot), dense(h0_dot), dense(c0_dot)
    w_dots = [dense(w) for w in w_dots]
    params = _lib.ptr_array([w.data_ptr() for w in weights])
    params_dot = _lib.ptr_array([ptr(w) for w in w_dots]) if any(w is not None for w in w_dots) else None
    with _on(dev):
        rc = lib.b200rnn_forward_tangent(
            ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params, y.data_ptr(), *ys,
            ptr(h_0), ptr(c_0), reserve.data_ptr(), None, ptr(x_dot), params_dot, ptr(h0_dot), ptr(c0_dot),
            y_dot.data_ptr(), *yds, h_n_dot.data_ptr(), ptr(c_n_dot), scratch.data_ptr(), _stream_ptr(dev))
    _lib.check(rc, "b200rnn_forward_tangent")
    return y_dot, h_n_dot, c_n_dot


def forward_ad_active(*tensors) -> bool:
    """Whether any of ``tensors`` is a dual tensor of the current ``torch.autograd.forward_ad`` level, whose tangent
    forward-mode AD will ask for (the model-shell fusions do not compute one, so they take their unfused expressions)"""
    if fwAD._current_level < 0:
        return False
    return any(t is not None and fwAD.unpack_dual(t).tangent is not None for t in tensors)


def check_forward_ad(cfg: RNNConfig, lengths) -> None:
    """The parts of the sequence path that have no forward mode raise here, before any launch"""
    if cfg.proj_size:
        raise _lib.B200RNNError("b200rnn: forward-mode AD (jvp / jacfwd / dual tensors) does not take proj_size")
    if cfg.dtype != torch.float32 or cfg.master_f32:
        raise _lib.B200RNNError("b200rnn: forward-mode AD (jvp / jacfwd / dual tensors) runs float32 modules outside "
                                "torch.autocast only")
    if lengths is not None:
        raise _lib.B200RNNError("b200rnn: forward-mode AD (jvp / jacfwd / dual tensors) does not take PackedSequence "
                                "input")


class _RNNFunction(torch.autograd.Function):
    """y, h_n[, c_n] = RNN(x, weights, h_0[, c_0]); x is the logical time-major view [T,B,I], h_0 / c_0 are None
    (zeros) or contiguous [L*D,B,HO] / [L*D,B,H] (HO = proj_size, or H without a projection). A projected LSTM always
    goes through the _hx entry points (with NULL states when hx is None): the _fused ones do not take proj_size."""

    # position of the first weight among forward()'s inputs (after ctx)
    _W0 = 8

    @staticmethod
    def forward(ctx, x_tm: torch.Tensor, cfg: RNNConfig, rng_state: Optional[torch.Tensor], grad_sink,
                lengths: Optional[torch.Tensor], save: bool, h_0: Optional[torch.Tensor], c_0: Optional[torch.Tensor],
                *weights: torch.Tensor):
        # `save` is decided by the caller: grad mode is always off in here, and needs_input_grad is True for
        # requires_grad weights even under torch.no_grad() (it would allocate the reserve and store gates for nothing).
        # SAVE_FOR_TANGENT: a dual input, whose tangent the jvp below computes from the reserve
        tangent = save == SAVE_FOR_TANGENT
        save = tangent or (bool(save) and any(ctx.needs_input_grad))
        y, h_n, c_n, reserve = _rnn_forward_impl(x_tm, cfg, rng_state, lengths, save, h_0, c_0, weights)
        if save:
            ctx.cfg = cfg
            ctx.grad_sink = grad_sink
            ctx.lengths = lengths
            ctx.save_for_backward(x_tm, y, reserve, h_0, c_0, *weights)
            if tangent:
                ctx.save_for_forward(x_tm, y, reserve, h_0, c_0, *weights)
        if c_n is None:
            return y, h_n
        return y, h_n, c_n

    @staticmethod
    def backward(ctx, dy, dh_n, dc_n=None):
        x_tm, y, reserve, h_0, c_0, *weights = ctx.saved_tensors
        # under a dual level, a dual output gradient or a dual saved input (x, a weight, h_0 / c_0) asks for the
        # gradient's own tangent, which the raw-pointer BPTT does not compute: refuse rather than drop it
        if forward_ad_active(dy, dh_n, dc_n, x_tm, h_0, c_0, *weights):
            raise _lib.B200RNNError("b200rnn: forward-over-reverse (a jvp of the recurrence's backward, e.g. a "
                                    "Hessian-vector product) is not supported")
        w0 = _RNNFunction._W0
        need = ctx.needs_input_grad
        dx, dh_0, dc_0, grads_out = _rnn_backward_impl(ctx.cfg, x_tm, y, reserve, h_0, c_0, weights, dy, dh_n, dc_n,
                                                       ctx.lengths, need[0], need[w0 - 2], need[w0 - 1], need[w0:],
                                                       ctx.grad_sink)
        return (dx, None, None, None, None, None, dh_0, dc_0, *grads_out)

    @staticmethod
    def jvp(ctx, x_dot, _cfg, _rng, _sink, _lengths, _save, h0_dot, c0_dot, *w_dots):
        """eager ``torch.autograd.forward_ad``: the tangent recurrence over the reserve the forward kept"""
        x_tm, y, reserve, h_0, c_0, *weights = ctx.saved_tensors
        y_dot, h_n_dot, c_n_dot = _func.tangent(ctx.cfg, x_tm, y, reserve, h_0, c_0, x_dot, h0_dot, c0_dot, weights,
                                                w_dots)
        return (y_dot, h_n_dot) if ctx.cfg.mode != _lib.LSTM else (y_dot, h_n_dot, c_n_dot)


class _LNRNNPoolFunction(torch.autograd.Function):
    """pooled[B, D*H] = sum over time of RNN(LayerNorm(x)) with everything around the encoder fused IN THE TRAINING
    GRAPH (SURVEY.md 8f rank 1): LayerNorm folded into the operand preparation of the layer-0 projection (forward) and
    run backwards inside ``b200rnn_backward_fused``; the time sum accumulated in the recurrence epilogue; and the pooled
    gradient broadcast over the steps inside the BPTT kernel - neither ``LN(x)`` as an autograd tensor nor the
    ``[T,B,D*H]`` output gradient ever exist. ``x.mean(dim=1)`` is this sum times 1/T (a [B,H] op left to autograd).
    """

    @staticmethod
    def forward(ctx, x_tm: torch.Tensor, cfg: RNNConfig, rng_state, grad_sink, ln_w, ln_b, ln_eps: float,
                *weights: torch.Tensor):
        lib = _lib.load()
        T, B, _ = x_tm.shape
        H, L, D = cfg.hidden_size, cfg.num_layers, cfg.num_dirs
        dev = x_tm.device
        fused_ln = ln_w is not None
        desc = _make_desc(cfg, B, T, True, fused_ln=fused_ln)
        rbytes, sbytes = _lib.workspace_bytes(desc)
        reserve = torch.empty(rbytes, dtype=torch.uint8, device=dev)
        scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
        y = torch.empty(T, B, D * H, dtype=torch.float32, device=dev)     # h_t of the top layer: BPTT needs h_{t-1}
        pooled = torch.empty(B, D * H, dtype=torch.float32, device=dev)
        h_n = torch.empty(L * D, B, H, dtype=torch.float32, device=dev)
        c_n = torch.empty(L * D, B, H, dtype=torch.float32, device=dev) if cfg.mode == _lib.LSTM else None
        params = _lib.ptr_array([w.data_ptr() for w in weights])
        with _on(dev):
            rc = lib.b200rnn_forward_fused(
                ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params,
                y.data_ptr(), B * D * H, D * H, h_n.data_ptr(), c_n.data_ptr() if c_n is not None else None,
                reserve.data_ptr(), scratch.data_ptr(), 0, 0,
                rng_state.data_ptr() if rng_state is not None else None,
                ln_w.data_ptr() if fused_ln else None, ln_b.data_ptr() if fused_ln else None, float(ln_eps),
                pooled.data_ptr(), None, None, None, _stream_ptr(dev))
        _lib.check(rc, "b200rnn_forward_fused")
        ctx.cfg, ctx.grad_sink, ctx.ln_eps, ctx.fused_ln = cfg, grad_sink, float(ln_eps), fused_ln
        ctx.save_for_backward(x_tm, y, reserve, ln_w if fused_ln else x_tm.new_empty(0), *weights)
        return pooled

    @staticmethod
    def backward(ctx, dpool):
        lib = _lib.load()
        cfg: RNNConfig = ctx.cfg
        x_tm, y, reserve, ln_w, *weights = ctx.saved_tensors
        T, B, I = x_tm.shape
        H, L, D = cfg.hidden_size, cfg.num_layers, cfg.num_dirs
        dev = x_tm.device
        dpool = dpool.contiguous()
        need_dx = ctx.needs_input_grad[0]
        dx = torch.empty(T, B, I, dtype=torch.float32, device=dev) if need_dx else None
        dln_w = torch.empty_like(ln_w) if (ctx.fused_ln and ctx.needs_input_grad[4]) else None
        dln_b = torch.empty_like(ln_w) if (ctx.fused_ln and ctx.needs_input_grad[5]) else None
        dptrs, grads_out, accumulate = _weight_grad_targets(weights, ctx.needs_input_grad[7:], ctx.grad_sink, dev)
        # with a sink the RNN weight gradients accumulate; the LayerNorm gradients are returned to autograd (fresh
        # tensors), so they must be WRITTEN: run them through a zeroed target when accumulating
        if accumulate:
            if dln_w is not None:
                dln_w.zero_()
            if dln_b is not None:
                dln_b.zero_()
        desc = _make_desc(cfg, B, T, True, accumulate, fused_ln=ctx.fused_ln)
        _, sbytes = _lib.workspace_bytes(desc)
        scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
        params = _lib.ptr_array([w.data_ptr() for w in weights])
        dparams = _lib.ptr_array(dptrs)
        with _on(dev):
            rc = lib.b200rnn_backward_fused(
                ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params,
                y.data_ptr(), B * D * H, D * H, None, 0, 0, dpool.data_ptr(), 1.0, None, None,
                reserve.data_ptr(), scratch.data_ptr(),
                dx.data_ptr() if dx is not None else None, B * I if dx is not None else 0, I if dx is not None else 0,
                dparams, None, ln_w.data_ptr() if ctx.fused_ln else None, ctx.ln_eps,
                dln_w.data_ptr() if dln_w is not None else None, dln_b.data_ptr() if dln_b is not None else None,
                _stream_ptr(dev))
        _lib.check(rc, "b200rnn_backward_fused")
        return (dx, None, None, None, dln_w, dln_b, None, *grads_out)


def rnn_ln_pool_sum(x: torch.Tensor, weights: Sequence[torch.Tensor], cfg: RNNConfig, rng_state=None, grad_sink=None,
                    ln_weight: Optional[torch.Tensor] = None, ln_bias: Optional[torch.Tensor] = None,
                    ln_eps: float = 1e-5) -> torch.Tensor:
    """``RNN(LayerNorm(x))[0].sum(dim=time)`` under autograd with the shell fused around the encoder (see
    :class:`_LNRNNPoolFunction`). ``x`` is [T,B,I] or [B,T,I] (``cfg.batch_first``); returns [B, D*H]."""
    _require_cuda_f32(x, "input")
    for i, w in enumerate(weights):
        _require_cuda_f32(w, f"weight[{i}]")
    if cfg.proj_size:
        raise NotImplementedError("b200rnn: the fused LayerNorm / time-sum path does not take proj_size")
    x_tm = _tm_view(x.transpose(0, 1) if cfg.batch_first else x)
    x_tm, ln_weight, ln_bias = _ln_operands(x_tm, ln_weight, ln_bias)
    return _LNRNNPoolFunction.apply(x_tm, cfg, rng_state, grad_sink, ln_weight, ln_bias, ln_eps, *weights)


def _initial_state(hx, cfg: RNNConfig, x: torch.Tensor):
    """(h_0, c_0) of ``hx`` - None, ``h_0`` (GRU) or ``(h_0, c_0)`` (LSTM) - checked as torch checks them (shapes:
    ``RNNBase.check_forward_args``, with its messages; then device and dtype against the input), contiguous. c_0 is
    None for the GRU; both are None without ``hx``."""
    if hx is None:
        return None, None
    lstm = cfg.mode == _lib.LSTM
    states = tuple(hx) if lstm else (hx,)
    if len(states) != (2 if lstm else 1):
        raise RuntimeError(f"b200rnn: LSTM hx must be a pair (h_0, c_0), got {len(states)} tensors")
    batch = x.size(0 if cfg.batch_first else 1) if x.dim() == 3 else None
    expected = [(cfg.num_layers * cfg.num_dirs, batch, w) for w in (cfg.out_size, cfg.hidden_size)]
    msgs = (("Expected hidden[0] size {}, got {}", "Expected hidden[1] size {}, got {}") if lstm
            else ("Expected hidden size {}, got {}",))
    for s, msg, want in zip(states, msgs, expected):
        if s.size() != want:
            raise RuntimeError(msg.format(want, list(s.size())))
    for s in states:
        if s.device != x.device:
            raise RuntimeError("Input and hidden tensors are not at the same device, found input tensor at "
                               f"{x.device} and hidden tensor at {s.device}")
        if s.dtype != x.dtype:
            raise RuntimeError("Input and hidden tensors are not the same dtype, found input tensor with "
                               f"{x.dtype} and hidden tensor with {s.dtype}")
    states = tuple(s.contiguous() for s in states)
    return states[0], (states[1] if lstm else None)


@torch.compiler.disable   # raised outside the trace, so that torch.compile hands the caller this error itself
def _grad_sink_untraceable():
    raise _lib.B200RNNError(
        "b200rnn: a module with a gradient sink (GradBucket / FlatAdamW) writes its gradients into the flat bucket "
        "behind autograd's back, which torch.compile and torch.export cannot trace; run it eagerly")


def rnn_forward(x: torch.Tensor, weights: Sequence[torch.Tensor], cfg: RNNConfig,
                rng_state: Optional[torch.Tensor] = None, grad_sink=None, lengths: Optional[torch.Tensor] = None,
                hx=None):
    """Run the multi-layer GRU / LSTM / Elman RNN. ``x`` is [T,B,I] (or [B,T,I] if ``cfg.batch_first``), any strides.

    ``hx`` is the initial state as torch takes it: None (zeros), ``h_0`` (GRU, RNN) or ``(h_0, c_0)`` (LSTM), each
    [L*D, B, H] with the rows in ``x``'s batch order (also with ``lengths``). It is differentiable: ``dh_0`` / ``dc_0``
    are computed only when autograd asks for them.

    Returns ``(y, h_n)`` for GRU and RNN and ``(y, h_n, c_n)`` for LSTM, laid out like torch.nn.GRU/LSTM/RNN outputs.
    """
    if cfg.dtype != torch.float32 and x.dtype != cfg.dtype:   # torch's check_input, before the state checks
        raise ValueError(f"RNN input dtype ({x.dtype}) does not match weight dtype ({cfg.dtype}). "
                         f"Convert input: input.to({cfg.dtype}), or convert model: model.to({x.dtype})")
    h_0, c_0 = _initial_state(hx, cfg, x)
    _require_cuda_dtype(x, "input", cfg.dtype)
    if x.dim() != 3:
        raise NotImplementedError("b200rnn: only batched 3-D input is supported (the reference never uses 2-D)")
    if cfg.dtype != torch.float32 and cfg.proj_size:
        raise NotImplementedError("b200rnn: proj_size is float32 only")
    for i, w in enumerate(weights):
        _require_cuda_dtype(w, f"weight[{i}]", torch.float32 if cfg.master_f32 else cfg.dtype)
        if not w.is_contiguous():
            raise _lib.B200RNNError(f"b200rnn: weight[{i}] must be contiguous")
    if x.size(2) != cfg.input_size:
        raise RuntimeError(f"input.size(-1) must be equal to input_size. Expected {cfg.input_size}, got {x.size(2)}")
    x_tm = x.transpose(0, 1) if cfg.batch_first else x
    x_tm = _tm_view(x_tm)
    if lengths is not None:
        lengths = lengths.to(device=x.device, dtype=torch.int32).contiguous()
    for i, w in enumerate(weights):
        if w.device != x.device:
            raise _lib.B200RNNError(f"b200rnn: weight[{i}] is on {w.device} but the input is on {x.device}")
    states = [s for s in (h_0, c_0) if s is not None]
    save = torch.is_grad_enabled() and (x.requires_grad or any(t.requires_grad for t in (*weights, *states)))
    if forward_ad_active(x, *weights, *states):   # a dual tensor: keep the reserve for the tangent recurrence
        check_forward_ad(cfg, lengths)
        save = SAVE_FOR_TANGENT
    if torch.compiler.is_compiling():   # dynamo / export: the custom op, which traces without a pointer
        if grad_sink is not None:
            _grad_sink_untraceable()
        return _ops.rnn_forward_traced(x_tm, cfg, rng_state, lengths, save, h_0, c_0, weights)
    if functorch_active():   # torch.func.grad / vmap / jvp: wrapped tensors have no pointer (b200rnn/func.py)
        _func.check_supported(cfg, lengths, grad_sink)
        return _func.rnn_forward(x_tm, cfg, rng_state, True, h_0, c_0, weights)
    return _RNNFunction.apply(x_tm, cfg, rng_state, grad_sink, lengths, save, h_0, c_0, *weights)


def functorch_active() -> bool:
    """Whether a torch.func transform (vmap, grad, ...) is running: its tensors have no data pointer, so the fused
    model-shell paths, which hand pointers to the library directly, are not taken"""
    return torch._C._are_functorch_transforms_active()


@torch.no_grad()
def rnn_forward_fused(x: torch.Tensor, weights: Sequence[torch.Tensor], cfg: RNNConfig,
                      rng_state: Optional[torch.Tensor] = None, ln_weight: Optional[torch.Tensor] = None,
                      ln_bias: Optional[torch.Tensor] = None, ln_eps: float = 1e-5, pool_sum: bool = False,
                      wcache: Optional[torch.Tensor] = None, prologue_done: Optional[torch.cuda.Event] = None):
    """No-grad forward with the shell fusions of ``b200rnn_forward_fused``: optional LayerNorm prologue on ``x``
    and, with ``pool_sum``, the sum over time of the output instead of the sequence (``[B, D*H]``).
    ``prologue_done`` is recorded on the current stream after the layer-0 operand preparation, before the first GEMM.

    Mirrors ``x = ln(x); x, _ = gru(x); x = x.sum(dim=1)`` (fuse_net_whole.py:360-362). Returns ``(out, h_n[, c_n])``.
    """
    lib = _lib.load()
    _require_cuda_f32(x, "input")
    if cfg.proj_size:
        raise NotImplementedError("b200rnn: the fused forward (LayerNorm prologue, time sum) does not take proj_size")
    x_tm = _tm_view(x.transpose(0, 1) if cfg.batch_first else x)
    x_tm, ln_weight, ln_bias = _ln_operands(x_tm, ln_weight, ln_bias)
    T, B, _ = x_tm.shape
    H, L, D = cfg.hidden_size, cfg.num_layers, cfg.num_dirs
    dev = x.device
    desc = _make_desc(cfg, B, T, False)
    _, sbytes = _lib.workspace_bytes(desc)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
    if pool_sum:
        out = torch.empty(B, D * H, dtype=torch.float32, device=dev)
        y_ptr, ys_t, ys_b, pool_ptr = None, 0, 0, out.data_ptr()
    elif cfg.batch_first:
        out = torch.empty(B, T, D * H, dtype=torch.float32, device=dev)
        y_ptr, ys_t, ys_b, pool_ptr = out.data_ptr(), D * H, T * D * H, None
    else:
        out = torch.empty(T, B, D * H, dtype=torch.float32, device=dev)
        y_ptr, ys_t, ys_b, pool_ptr = out.data_ptr(), B * D * H, D * H, None
    h_n = torch.empty(L * D, B, H, dtype=torch.float32, device=dev)
    c_n = torch.empty(L * D, B, H, dtype=torch.float32, device=dev) if cfg.mode == _lib.LSTM else None
    params = _lib.ptr_array([w.data_ptr() for w in weights])
    if prologue_done is not None and not prologue_done.cuda_event:
        prologue_done.record()      # torch creates the CUDA event at its first record
    with _on(dev):
        rc = lib.b200rnn_forward_fused(
            ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params, y_ptr, ys_t, ys_b,
            h_n.data_ptr(), c_n.data_ptr() if c_n is not None else None, None, scratch.data_ptr(), 0, 0,
            rng_state.data_ptr() if rng_state is not None else None,
            ln_weight.data_ptr() if ln_weight is not None else None,
            ln_bias.data_ptr() if ln_bias is not None else None,
            float(ln_eps), pool_ptr, None, wcache.data_ptr() if wcache is not None else None,
            prologue_done.cuda_event if prologue_done is not None else None, _stream_ptr(dev))
    _lib.check(rc, "b200rnn_forward_fused")
    return (out, h_n) if c_n is None else (out, h_n, c_n)


def prepare_weights(weights: Sequence[torch.Tensor], cfg: RNNConfig) -> torch.Tensor:
    """TF32 hi/lo and fp16-pair splits of every ``weight_ih`` and, for a unidirectional GRU-256, the fp16 pairs of
    every ``weight_hh`` (``b200rnn_prepare_weights``): the weight cache ``rnn_forward_fused`` accepts so that frozen
    encoders split their weights once instead of once per step."""
    lib = _lib.load()
    dev = weights[0].device
    for i, w in enumerate(weights):
        _require_cuda_f32(w, f"weight[{i}]")
    desc = _make_desc(cfg, 1, 1, False)
    n = ctypes.c_size_t(0)
    _lib.check(lib.b200rnn_wcache_bytes(ctypes.byref(desc), ctypes.byref(n)), "b200rnn_wcache_bytes")
    cache = torch.empty(int(n.value), dtype=torch.uint8, device=dev)
    params = _lib.ptr_array([w.data_ptr() for w in weights])
    with _on(dev):
        rc = lib.b200rnn_prepare_weights(ctypes.byref(desc), params, cache.data_ptr(), _stream_ptr(dev))
    _lib.check(rc, "b200rnn_prepare_weights")
    return cache


@dataclass
class CellConfig:
    mode: int            # _lib.GRU / _lib.LSTM / _lib.RNN_TANH / _lib.RNN_RELU
    input_size: int
    hidden_size: int
    bias: bool
    tf32: bool = False   # single-pass TF32 contraction and gradient GEMMs (tf32_enabled()), else 3xTF32


def _cell_desc(cfg: CellConfig, B: int, save: bool) -> _lib.CellDesc:
    flags = _lib.FLAG_SAVE_FOR_BACKWARD if save else 0
    if cfg.tf32:
        flags |= _lib.FLAG_TF32
    if not cfg.bias:
        flags |= _lib.FLAG_NO_BIAS
    return _lib.CellDesc(cfg.mode, B, cfg.input_size, cfg.hidden_size, flags)


def _cell_rows(t: torch.Tensor) -> torch.Tensor:
    """``t`` [R, C] as the cell entry points take it: feature stride 1 and rows that do not overlap (copy if not)"""
    if (t.stride(1) != 1 and t.size(1) != 1) or (t.size(0) > 1 and t.stride(0) < t.size(1)):
        t = t.contiguous()
    return t


def _cell_forward_buffers(x: torch.Tensor, cfg: CellConfig, save: bool):
    """``(desc, saved, h_out, c_out)`` of one cell forward (``c_out`` None but for the LSTM, ``saved`` empty without
    ``save``): host arithmetic only, shared with the ``b200rnn::cell_forward`` op's fake implementation"""
    B, H, dev = x.size(0), cfg.hidden_size, x.device
    desc = _cell_desc(cfg, B, save)
    sv_bytes, _ = _lib.cell_workspace_bytes(desc)
    saved = torch.empty(sv_bytes if save else 0, dtype=torch.uint8, device=dev)
    h_out = torch.empty(B, H, dtype=torch.float32, device=dev)
    c_out = torch.empty(B, H, dtype=torch.float32, device=dev) if cfg.mode == _lib.LSTM else None
    return desc, saved, h_out, c_out


def _cell_forward_impl(x, cfg: CellConfig, save: bool, h, c, weights):
    """one ``b200rnn_cell_forward`` call, shared by :class:`_CellFunction` and the ``b200rnn::cell_forward`` op:
    returns ``(h_out, c_out, saved)``"""
    lib = _lib.load()
    dev = x.device
    desc, saved, h_out, c_out = _cell_forward_buffers(x, cfg, save)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    ld = lambda t: t.stride(0) if t is not None else 0  # noqa: E731
    params = _lib.ptr_array([w.data_ptr() for w in weights] + [None] * (4 - len(weights)))
    with _on(dev):
        rc = lib.b200rnn_cell_forward(ctypes.byref(desc), x.data_ptr(), x.stride(0), ptr(h), ld(h), ptr(c), ld(c),
                                      params, h_out.data_ptr(), ptr(c_out), saved.data_ptr() if save else None,
                                      _stream_ptr(dev))
    _lib.check(rc, "b200rnn_cell_forward")
    return h_out, c_out, saved


def _cell_grad_buffers(x, cfg: CellConfig, h, c, need_dx: bool, need_dh: bool, need_dc: bool):
    """``(dx, dh, dc)`` of a cell backward, None where not wanted"""
    B, I, H, dev = x.size(0), cfg.input_size, cfg.hidden_size, x.device
    new = lambda n: torch.empty(B, n, dtype=torch.float32, device=dev)  # noqa: E731
    dx = new(I) if need_dx else None
    dh = new(H) if h is not None and need_dh else None
    dc = new(H) if c is not None and need_dc else None
    return dx, dh, dc


def _cell_backward_impl(cfg: CellConfig, x, h, c, saved, weights, dh_out, dc_out, need_dx: bool, need_dh: bool,
                        need_dc: bool, need_w, separate: bool = False):
    """one ``b200rnn_cell_backward`` call, shared by :class:`_CellFunction` and the ``b200rnn::cell_backward`` op:
    returns ``(dx, dh, dc, weight grads)``, None for every gradient that is not wanted"""
    lib = _lib.load()
    B, dev = x.size(0), x.device
    dx, dh, dc = _cell_grad_buffers(x, cfg, h, c, need_dx, need_dh, need_dc)
    dptrs, grads_out, _ = _weight_grad_targets(weights, need_w, None, dev, separate)
    desc = _cell_desc(cfg, B, True)
    _, sbytes = _lib.cell_workspace_bytes(desc)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
    dh_out = dh_out.contiguous() if dh_out is not None else None
    dc_out = dc_out.contiguous() if dc_out is not None else None
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    ld = lambda t: t.stride(0) if t is not None else 0  # noqa: E731
    params = _lib.ptr_array([w.data_ptr() for w in weights] + [None] * (4 - len(weights)))
    dparams = _lib.ptr_array(dptrs + [None] * (4 - len(dptrs)))
    with _on(dev):
        rc = lib.b200rnn_cell_backward(ctypes.byref(desc), x.data_ptr(), x.stride(0), ptr(h), ld(h), ptr(c), ld(c),
                                       params, ptr(dh_out), ptr(dc_out), saved.data_ptr(), ptr(dx), ptr(dh),
                                       ptr(dc), dparams, scratch.data_ptr(), _stream_ptr(dev))
    _lib.check(rc, "b200rnn_cell_backward")
    return dx, dh, dc, grads_out


class _CellFunction(torch.autograd.Function):
    """h' (GRU) or (h', c') (LSTM) = cell(x, h, c, weights) for x [B, I]; h / c are None (zeros) or [B, H]. The TF32
    mode is in ``cfg``, read once per call, and the backward reuses it."""

    # position of the first weight among forward()'s inputs (after ctx)
    _W0 = 5

    @staticmethod
    def forward(ctx, x: torch.Tensor, cfg: CellConfig, save: bool, h: Optional[torch.Tensor],
                c: Optional[torch.Tensor], *weights: torch.Tensor):
        # as in _RNNFunction: the caller decides from grad mode, needs_input_grad confirms
        save = bool(save) and any(ctx.needs_input_grad)
        h_out, c_out, saved = _cell_forward_impl(x, cfg, save, h, c, weights)
        if save:
            ctx.cfg = cfg
            ctx.save_for_backward(x, h, c, saved, *weights)
        return h_out if c_out is None else (h_out, c_out)

    @staticmethod
    def backward(ctx, dh_out, dc_out=None):
        x, h, c, saved, *weights = ctx.saved_tensors
        need = ctx.needs_input_grad
        w0 = _CellFunction._W0
        dx, dh, dc, grads_out = _cell_backward_impl(ctx.cfg, x, h, c, saved, weights, dh_out, dc_out, need[0],
                                                    need[w0 - 2], need[w0 - 1], need[w0:])
        return (dx, None, None, dh, dc, *grads_out)


def cell_forward(x: torch.Tensor, hx, weights: Sequence[torch.Tensor], cfg: CellConfig, name: str):
    """One GRUCell / LSTMCell / RNNCell step on batched input: ``x`` [B, I], ``hx`` None (zeros), ``h`` (GRU, RNN) or ``(h, c)``
    (LSTM), each [B, H]; ``weights`` = (weight_ih, weight_hh[, bias_ih, bias_hh]). Shapes are checked as torch's
    ``_VF.gru_cell`` / ``_VF.lstm_cell`` check them (same exception types and messages), before the missing CPU path.
    Returns ``h'`` or ``(h', c')``."""
    lstm = cfg.mode == _lib.LSTM
    states = ()
    if hx is not None:
        if lstm and not isinstance(hx, (tuple, list)):
            raise TypeError(f"lstm_cell(): argument 'hx' (position 2) must be tuple of Tensors, not {type(hx).__name__}")
        states = tuple(hx) if lstm else (hx,)
        if lstm and len(states) != 2:
            raise RuntimeError("lstm_cell expects two hidden states")
    if x.size(1) != cfg.input_size:
        raise RuntimeError(f"input has inconsistent input_size: got {x.size(1)} expected {cfg.input_size}")
    for idx, s in enumerate(states):
        if s.size(0) != x.size(0):
            raise RuntimeError(f"Input batch size {x.size(0)} doesn't match hidden{idx} batch size {s.size(0)}")
        if s.size(1) != cfg.hidden_size:
            raise RuntimeError(f"hidden{idx} has inconsistent hidden_size: got {s.size(1)}, expected {cfg.hidden_size}")
    for s in states:
        if s.device != x.device:
            raise RuntimeError("Input and hidden tensors are not at the same device, found input tensor at "
                               f"{x.device} and hidden tensor at {s.device}")
        if s.dtype != x.dtype:
            raise RuntimeError("Input and hidden tensors are not the same dtype, found input tensor with "
                               f"{x.dtype} and hidden tensor with {s.dtype}")
    _require_cuda_f32(x, "input")
    for w in weights:
        _require_cuda_f32(w, f"{name} weight")
        if not w.is_contiguous():
            raise _lib.B200RNNError(f"b200rnn: {name} weights must be contiguous")
        if w.device != x.device:
            raise _lib.B200RNNError(f"b200rnn: a {name} weight is on {w.device} but the input is on {x.device}")
    x = _cell_rows(x)
    states = tuple(_cell_rows(s) for s in states)
    h, c = (states + (None, None))[:2]
    save = torch.is_grad_enabled() and (x.requires_grad or any(t.requires_grad for t in (*weights, *states)))
    if torch.compiler.is_compiling():
        return _ops.cell_forward_traced(x, cfg, save, h, c, weights)
    return _CellFunction.apply(x, cfg, save, h, c, *weights)


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_kcontig: bool = True, b_kcontig: bool = True,
         bias: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, accumulate: bool = False,
         use_splitk: bool = True) -> torch.Tensor:
    """C = A(m,k) B(k,n) (+bias) through ``b200rnn_gemm_f32`` — exposed for the parity tests.

    a: [M,K] if a_kcontig else [K,M];  b: [N,K] if b_kcontig else [K,N]; row-major, last stride 1.
    """
    lib = _lib.load()
    _require_cuda_f32(a, "a")
    _require_cuda_f32(b, "b")
    M, K = (a.shape if a_kcontig else (a.shape[1], a.shape[0]))
    N = b.shape[0] if b_kcontig else b.shape[1]
    Kb = b.shape[1] if b_kcontig else b.shape[0]
    assert K == Kb, (a.shape, b.shape)
    assert (a.stride(1) == 1 or a.size(1) == 1) and (b.stride(1) == 1 or b.size(1) == 1)
    lda = a.stride(0) if a.size(1) > 1 else 1
    ldb = b.stride(0) if b.size(1) > 1 else 1
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=a.device)
        assert not accumulate
    sbytes = max(M * N * 4 * 64, 8 * (M + N) * K + 4096) if use_splitk else 0
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=a.device) if sbytes else None
    with _on(a.device):
        rc = lib.b200rnn_gemm_f32(M, N, K, a.data_ptr(), lda, int(a_kcontig), b.data_ptr(), ldb,
                                  int(b_kcontig), out.data_ptr(), out.stride(0),
                                  bias.data_ptr() if bias is not None else None, int(accumulate),
                                  scratch.data_ptr() if scratch is not None else None, sbytes, _stream_ptr(a.device))
    _lib.check(rc, "b200rnn_gemm_f32")
    return out


# the custom ops (b200rnn/ops.py) and the torch.func path (b200rnn/func.py) wrap the helpers above; imported last
# because they import this module
from . import func as _func  # noqa: E402
from . import ops as _ops  # noqa: E402
