"""The sequence and cell entry points as ``torch.library`` custom ops, namespace ``b200rnn``.

``torch.export``, dynamo and AOTAutograd trace through FakeTensors, which have no ``data_ptr()``, so they cannot run the
``torch.autograd.Function`` bridges of :mod:`b200rnn.functional`. Under ``torch.compiler.is_compiling()``
``functional.rnn_forward`` and ``functional.cell_forward`` call these ops instead, after the same argument checks:

* ``b200rnn::rnn_forward`` / ``b200rnn::rnn_backward``: the multi-layer GRU / LSTM / Elman RNN and its BPTT;
* ``b200rnn::cell_forward`` / ``b200rnn::cell_backward``: one GRUCell / LSTMCell / RNNCell step and its gradient.

The CUDA implementations are the bodies of ``_RNNFunction`` / ``_CellFunction`` (the same library calls, buffers and
workspace sizes). The fake implementations allocate the same outputs through the same helpers and size the reserve
with ``b200rnn_workspace_bytes``, which is host arithmetic, so fake and real shapes agree by construction; they launch
nothing and read no pointer. The forward declares ``rng_state`` (the module's Philox ``{seed, offset}``) mutated: the
kernels advance its offset in place, and functionalization and CUDA-graph trees must carry that write.

Every output exists in every call so that the schemas have fixed arity: ``c_n`` / ``c_out`` is an empty ``[0]`` tensor
for the GRU and the Elman RNN, and so is every gradient the ``needs`` list does not ask for. Eager calls keep the
``autograd.Function`` path; the ops are what an exported program calls.
"""
from typing import List, Optional, Sequence, Tuple

import torch
from torch import Tensor

from . import _lib
from . import functional as F


def _rnn_config(kind, input_size, hidden_size, num_layers, num_dirs, proj_size, dropout, training, batch_first, tf32,
                dtype, weights) -> F.RNNConfig:
    """``master_f32`` (fp32 master parameters of a 16-bit call, ``torch.autocast``) is not an attribute of the ops: it
    is what fp32 ``weights`` beside a 16-bit ``dtype`` mean, so the schemas stay as they were"""
    master_f32 = dtype != torch.float32 and len(weights) > 0 and weights[0].dtype == torch.float32
    return F.RNNConfig(mode=kind, input_size=input_size, hidden_size=hidden_size, num_layers=num_layers,
                       num_dirs=num_dirs, dropout=dropout, training=training, batch_first=batch_first, tf32=tf32,
                       proj_size=proj_size, dtype=dtype, master_f32=master_f32)


def _rnn_attrs(cfg: F.RNNConfig) -> tuple:
    """the plain attributes of the rnn ops, in schema order"""
    return (cfg.mode, cfg.input_size, cfg.hidden_size, cfg.num_layers, cfg.num_dirs, cfg.proj_size, float(cfg.dropout),
            bool(cfg.training), bool(cfg.batch_first), bool(cfg.tf32), cfg.dtype)


def _none(t: Optional[Tensor], like: Tensor) -> Tensor:
    """``t``, or the empty ``[0]`` stand-in for an output that does not exist in this call"""
    return t if t is not None else like.new_empty(0)


def _some(t: Tensor, wanted: bool) -> Optional[Tensor]:
    return t if wanted else None


# -- sequence ------------------------------------------------------------------------------------------------------

# rnn_forward mutates rng_state, and torch.library.custom_op takes an autograd formula only for functional ops, so
# this one op is defined with the low-level API: schema, CUDA kernel, fake kernel and an Autograd kernel that wraps
# the call below autograd in an autograd.Function (the structure custom_op builds for a functional op).
_DEF = torch.library.Library("b200rnn", "FRAGMENT")
_DEF.define(
    "rnn_forward(Tensor x, Tensor[] weights, Tensor? h_0, Tensor? c_0, Tensor? lengths, Tensor(a!)? rng_state, "
    "int kind, int input_size, int hidden_size, int num_layers, int num_dirs, int proj_size, float dropout, "
    "bool training, bool batch_first, bool tf32, ScalarType dtype, bool save) -> (Tensor, Tensor, Tensor, Tensor)")


def _rnn_forward_cuda(x, weights, h_0, c_0, lengths, rng_state, kind, input_size, hidden_size, num_layers, num_dirs,
                      proj_size, dropout, training, batch_first, tf32, dtype, save):
    """``(y, h_n, c_n, reserve)`` of the RNN over the time-major view ``x`` [T, B, I]; the reserve (uint8) holds what
    the backward reads and is empty without ``save``."""
    cfg = _rnn_config(kind, input_size, hidden_size, num_layers, num_dirs, proj_size, dropout, training, batch_first,
                      tf32, dtype, weights)
    y, h_n, c_n, reserve = F._rnn_forward_impl(x, cfg, rng_state, lengths, save, h_0, c_0, weights)
    return y, h_n, _none(c_n, y), reserve


def _rnn_forward_fake(x, weights, h_0, c_0, lengths, rng_state, kind, input_size, hidden_size, num_layers, num_dirs,
                      proj_size, dropout, training, batch_first, tf32, dtype, save):
    cfg = _rnn_config(kind, input_size, hidden_size, num_layers, num_dirs, proj_size, dropout, training, batch_first,
                      tf32, dtype, weights)
    _, reserve, _, y, _, h_n, c_n = F._forward_buffers(x, cfg, save, with_scratch=False)
    return y, h_n, _none(c_n, y), reserve


class _RNNForwardAutograd(torch.autograd.Function):
    """autograd of ``b200rnn::rnn_forward``: saves what ``_RNNFunction`` saves, differentiates through
    ``b200rnn::rnn_backward``"""

    @staticmethod
    def forward(ctx, x, h_0, c_0, lengths, rng_state, attrs, save, *weights):
        with torch._C._AutoDispatchBelowADInplaceOrView():
            y, h_n, c_n, reserve = torch.ops.b200rnn.rnn_forward.default(x, list(weights), h_0, c_0, lengths,
                                                                         rng_state, *attrs, save)
        ctx.mark_non_differentiable(reserve)
        ctx.attrs = attrs
        ctx.save_for_backward(x, y, reserve, h_0, c_0, lengths, *weights)
        return y, h_n, c_n, reserve

    @staticmethod
    def backward(ctx, dy, dh_n, dc_n, _dreserve):
        x, y, reserve, h_0, c_0, lengths, *weights = ctx.saved_tensors
        need = ctx.needs_input_grad
        needs = [bool(need[0]), h_0 is not None and bool(need[1]), c_0 is not None and bool(need[2]),
                 *map(bool, need[7:])]
        lstm = ctx.attrs[0] == _lib.LSTM
        dx, dh_0, dc_0, dws = rnn_backward(x, y, reserve, h_0, c_0, weights, dy, dh_n, dc_n if lstm else None,
                                           lengths, needs, *ctx.attrs)
        return (_some(dx, needs[0]), _some(dh_0, needs[1]), _some(dc_0, needs[2]), None, None, None, None,
                *(_some(g, n) for g, n in zip(dws, needs[3:])))


def _rnn_forward_autograd(x, weights, h_0, c_0, lengths, rng_state, *attrs_save):
    return _RNNForwardAutograd.apply(x, h_0, c_0, lengths, rng_state, attrs_save[:-1], attrs_save[-1], *weights)


_DEF.impl("rnn_forward", _rnn_forward_cuda, "CUDA")
_DEF.impl("rnn_forward", _rnn_forward_autograd, "Autograd")
torch.library.register_fake("b200rnn::rnn_forward", _rnn_forward_fake, lib=_DEF)


@torch.library.custom_op("b200rnn::rnn_backward", mutates_args=(), device_types="cuda")
def rnn_backward(x: Tensor, y: Tensor, reserve: Tensor, h_0: Optional[Tensor], c_0: Optional[Tensor],
                 weights: List[Tensor], dy: Optional[Tensor], dh_n: Optional[Tensor], dc_n: Optional[Tensor],
                 lengths: Optional[Tensor], needs: List[bool], kind: int, input_size: int, hidden_size: int,
                 num_layers: int, num_dirs: int, proj_size: int, dropout: float, training: bool, batch_first: bool,
                 tf32: bool, dtype: torch.dtype) -> Tuple[Tensor, Tensor, Tensor, List[Tensor]]:
    """``(dx, dh_0, dc_0, weight grads)``. ``needs`` = [dx, dh_0, dc_0, one per weight]: what is not needed is not
    computed (a NULL pointer to the library) and comes back as an empty ``[0]`` tensor."""
    cfg = _rnn_config(kind, input_size, hidden_size, num_layers, num_dirs, proj_size, dropout, training, batch_first,
                      tf32, dtype, weights)
    dx, dh_0, dc_0, dws = F._rnn_backward_impl(cfg, x, y, reserve, h_0, c_0, weights, dy, dh_n, dc_n, lengths,
                                               needs[0], needs[1], needs[2], needs[3:], None, separate=True)
    return _none(dx, x), _none(dh_0, x), _none(dc_0, x), [_none(g, w) for g, w in zip(dws, weights)]


@rnn_backward.register_fake
def _rnn_backward_fake(x, y, reserve, h_0, c_0, weights, dy, dh_n, dc_n, lengths, needs, kind, input_size,
                       hidden_size, num_layers, num_dirs, proj_size, dropout, training, batch_first, tf32, dtype):
    dx = F._dx_buffer(x) if needs[0] else None
    dh_0 = torch.empty_like(h_0) if h_0 is not None and needs[1] else None
    dc_0 = torch.empty_like(c_0) if c_0 is not None and needs[2] else None
    dws = F._weight_grad_buffers(weights, needs[3:])
    return _none(dx, x), _none(dh_0, x), _none(dc_0, x), [_none(g, w) for g, w in zip(dws, weights)]


def rnn_forward_traced(x_tm: Tensor, cfg: F.RNNConfig, rng_state: Optional[Tensor], lengths: Optional[Tensor],
                       save: bool, h_0: Optional[Tensor], c_0: Optional[Tensor], weights: Sequence[Tensor]):
    """``_RNNFunction.apply`` through the op: ``(y, h_n)``, or ``(y, h_n, c_n)`` for the LSTM"""
    y, h_n, c_n, _ = torch.ops.b200rnn.rnn_forward(x_tm, list(weights), h_0, c_0, lengths, rng_state, *_rnn_attrs(cfg), bool(save))
    return (y, h_n, c_n) if cfg.mode == _lib.LSTM else (y, h_n)


# -- cells ---------------------------------------------------------------------------------------------------------

def _cell_config(kind, input_size, hidden_size, bias, tf32) -> F.CellConfig:
    return F.CellConfig(mode=kind, input_size=input_size, hidden_size=hidden_size, bias=bias, tf32=tf32)


@torch.library.custom_op("b200rnn::cell_forward", mutates_args=(), device_types="cuda")
def cell_forward(x: Tensor, h: Optional[Tensor], c: Optional[Tensor], weights: List[Tensor], kind: int,
                 input_size: int, hidden_size: int, bias: bool, tf32: bool, save: bool) -> Tuple[Tensor, Tensor, Tensor]:
    """``(h_out, c_out, saved)`` of one cell step on ``x`` [B, I]; ``saved`` (uint8) is empty without ``save``."""
    cfg = _cell_config(kind, input_size, hidden_size, bias, tf32)
    h_out, c_out, saved = F._cell_forward_impl(x, cfg, save, h, c, weights)
    return h_out, _none(c_out, h_out), saved


@cell_forward.register_fake
def _cell_forward_fake(x, h, c, weights, kind, input_size, hidden_size, bias, tf32, save):
    _, saved, h_out, c_out = F._cell_forward_buffers(x, _cell_config(kind, input_size, hidden_size, bias, tf32), save)
    return h_out, _none(c_out, h_out), saved


@torch.library.custom_op("b200rnn::cell_backward", mutates_args=(), device_types="cuda")
def cell_backward(x: Tensor, h: Optional[Tensor], c: Optional[Tensor], saved: Tensor, weights: List[Tensor],
                  dh_out: Optional[Tensor], dc_out: Optional[Tensor], needs: List[bool], kind: int, input_size: int,
                  hidden_size: int, bias: bool, tf32: bool) -> Tuple[Tensor, Tensor, Tensor, List[Tensor]]:
    """``(dx, dh, dc, weight grads)``; ``needs`` = [dx, dh, dc, one per weight], as in ``rnn_backward``."""
    cfg = _cell_config(kind, input_size, hidden_size, bias, tf32)
    dx, dh, dc, dws = F._cell_backward_impl(cfg, x, h, c, saved, weights, dh_out, dc_out, needs[0], needs[1],
                                            needs[2], needs[3:], separate=True)
    return _none(dx, x), _none(dh, x), _none(dc, x), [_none(g, w) for g, w in zip(dws, weights)]


@cell_backward.register_fake
def _cell_backward_fake(x, h, c, saved, weights, dh_out, dc_out, needs, kind, input_size, hidden_size, bias, tf32):
    cfg = _cell_config(kind, input_size, hidden_size, bias, tf32)
    dx, dh, dc = F._cell_grad_buffers(x, cfg, h, c, needs[0], needs[1], needs[2])
    dws = F._weight_grad_buffers(weights, needs[3:])
    return _none(dx, x), _none(dh, x), _none(dc, x), [_none(g, w) for g, w in zip(dws, weights)]


def _cell_setup_context(ctx, inputs, output):
    x, h, c, weights, *attrs = inputs
    ctx.attrs = attrs[:-1]   # without `save`
    ctx.save_for_backward(x, h, c, output[2], *weights)


def _cell_backward_formula(ctx, dh_out, dc_out, _dsaved):
    x, h, c, saved, *weights = ctx.saved_tensors
    need_x, need_h, need_c, need_w = ctx.needs_input_grad[:4]
    needs = [bool(need_x), h is not None and bool(need_h), c is not None and bool(need_c), *map(bool, need_w)]
    lstm = ctx.attrs[0] == _lib.LSTM
    dx, dh, dc, dws = cell_backward(x, h, c, saved, weights, dh_out, dc_out if lstm else None, needs, *ctx.attrs)
    dws = [_some(g, n) for g, n in zip(dws, needs[3:])]
    return (_some(dx, needs[0]), _some(dh, needs[1]), _some(dc, needs[2]), dws, *([None] * (len(ctx.attrs) + 1)))


cell_forward.register_autograd(_cell_backward_formula, setup_context=_cell_setup_context)


def cell_forward_traced(x: Tensor, cfg: F.CellConfig, save: bool, h: Optional[Tensor], c: Optional[Tensor],
                        weights: Sequence[Tensor]):
    """``_CellFunction.apply`` through the op: ``h'``, or ``(h', c')`` for the LSTM"""
    h_out, c_out, _ = cell_forward(x, h, c, list(weights), cfg.mode, cfg.input_size, cfg.hidden_size, bool(cfg.bias),
                                   bool(cfg.tf32), bool(save))
    return (h_out, c_out) if cfg.mode == _lib.LSTM else h_out
