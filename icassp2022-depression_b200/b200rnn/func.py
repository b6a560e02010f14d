"""The sequence entry point under ``torch.func`` transforms: ``grad`` / ``grad_and_value`` / ``vjp`` and ``vmap``.

The eager bridge (``functional._RNNFunction``) hands raw pointers to the library, and functorch's wrapped tensors have
none. Inside any functorch transform ``functional.rnn_forward`` therefore calls :func:`rnn_forward` here: an
``autograd.Function`` in the form torch.func composes with (``setup_context`` and ``vmap`` staticmethods), whose
forward and backward are the eager ones. (A custom op's registered autograd formula does not run under
``torch.func.grad`` in torch 2.11, so this path does not go through the ``b200rnn::rnn_forward`` op.)

``vmap`` over M models (``torch.func.stack_module_state`` + ``functional_call``), or over M samples for per-sample
gradients, is one library call for all of them (``RNNConfig.models``): each recurrence layer runs every model in one
launch of the runtime-sized cluster kernels, forward and backward, and the GEMMs run per model. A tensor the vmap
does not batch (shared weights, a shared ``x``) is passed with model stride 0 and not copied; an unbatched ``hx`` is
expanded into a dense block. Inter-layer dropout follows vmap's ``randomness``: ``'error'`` raises what
``torch.nn.functional.dropout`` raises; ``'different'`` takes model m's mask from row m of a batched ``_rng_state``, or,
from an unbatched one, the mask the m-th of M consecutive one-model calls would draw; ``'same'`` applies one mask to
every model and needs an unbatched state. Each state advances as the Python loop over the models would advance it.

Forward mode: ``torch.func.jvp`` / ``jacfwd`` (and eager ``torch.autograd.forward_ad`` dual tensors, through
``functional._RNNFunction.jvp``) compute the tangent with :class:`_Tangent`, one ``b200rnn_forward_tangent`` call over the
reserve the forward kept: the tangent pre-activations by the time-parallel GEMMs, then one tangent recurrence launch per
layer. ``jacfwd`` vmaps the jvp over M tangent directions: :meth:`_Tangent.vmap` passes them to the library as one call,
each recurrence layer running all M in one launch, the primal shared. Second-order products (``hessian``,
``jvp(grad(f))``, the gradient of a tangent) raise ``B200RNNError``.

The one call is not always the faster one (README, tools/ensemble_steps_results.json): it wins for small batches from a
handful of models on and for per-sample gradients, and loses for one model (the transform's host cost) and for large
batches at hidden sizes 128 / 256, where a loop runs the fixed configs tuned for them and the ensemble the
runtime-sized kernels.
"""
from __future__ import annotations

import dataclasses
from typing import Optional, Sequence

import torch

from . import _lib
from . import functional as F

_RANDOMNESS_ERROR = ("vmap: called random operation while in randomness error mode. Please either use the 'same' or "
                     "'different' randomness flags on vmap or perform the randomness operation out of vmap")


def check_supported(cfg: F.RNNConfig, lengths, grad_sink) -> None:
    """The parts of the sequence path that do not run under a functorch transform raise here, before any launch."""
    if cfg.proj_size:
        raise _lib.B200RNNError("b200rnn: proj_size does not run under torch.func transforms (vmap / grad)")
    if cfg.dtype != torch.float32 or cfg.master_f32:
        raise _lib.B200RNNError("b200rnn: torch.func transforms (vmap / grad) run float32 modules outside "
                                "torch.autocast only")
    if lengths is not None:
        raise _lib.B200RNNError("b200rnn: PackedSequence input does not run under torch.func transforms (vmap / grad)")
    if grad_sink is not None:
        raise _lib.B200RNNError("b200rnn: a module with a gradient sink (GradBucket / FlatAdamW) writes its gradients "
                                "behind autograd's back, which torch.func transforms cannot follow")


def _to_models(t: Optional[torch.Tensor], bdim: Optional[int], M: int, dense: bool) -> Optional[torch.Tensor]:
    """``t`` with its vmap dimension first, [M, ...]; an unbatched tensor expanded (model stride 0) or, ``dense``,
    copied into a dense block"""
    if t is None:
        return None
    t = t.movedim(bdim, 0) if bdim is not None else t.expand(M, *t.shape)
    return t.contiguous() if dense else t


def _one_model(ts, M: int):
    """with M = 1 the call is the one-model call: each [1, ...] tensor without its model dimension"""
    return [t[0] if M == 1 and t is not None else t for t in ts]


def _with_model_dim(outs, out_dims, M: int):
    """the outputs of a call made by :func:`_one_model`, with the model dimension put back"""
    return tuple(o.unsqueeze(0) if M == 1 and d == 0 else o for o, d in zip(outs, out_dims))


def _weight_models(w: torch.Tensor, bdim: Optional[int], M: int) -> torch.Tensor:
    """a parameter as the library reads M of them: [M, ...] with each model's block contiguous, stride 0 if shared"""
    w = _to_models(w, bdim, M, dense=False)
    if w.stride(0) != 0 and not w.is_contiguous():
        w = w.contiguous()
    return w


class _Forward(torch.autograd.Function):
    """``(y, h_n, c_n, reserve)`` of the sequence forward over the time-major ``x_tm``; ``c_n`` is an empty stand-in but
    for the LSTM, ``reserve`` is empty without ``save``"""

    @staticmethod
    def forward(x_tm, cfg, rng_state, save, h_0, c_0, *weights):
        y, h_n, c_n, reserve = F._rnn_forward_impl(x_tm, cfg, rng_state, None, save, h_0, c_0, weights)
        return y, h_n, c_n if c_n is not None else y.new_empty(0), reserve

    @staticmethod
    def setup_context(ctx, inputs, output):
        x_tm, cfg, _, save, h_0, c_0, *weights = inputs
        y, _, c_n, reserve = output
        ctx.mark_non_differentiable(reserve)
        if cfg.mode != _lib.LSTM:
            ctx.mark_non_differentiable(c_n)
        ctx.cfg = cfg
        if save:
            ctx.save_for_backward(x_tm, y, reserve, h_0, c_0, *weights)
            ctx.save_for_forward(x_tm, y, reserve, h_0, c_0, *weights)

    @staticmethod
    def backward(ctx, dy, dh_n, dc_n, _dreserve):
        x_tm, y, reserve, h_0, c_0, *weights = ctx.saved_tensors
        need = ctx.needs_input_grad
        needs = (bool(need[0]), h_0 is not None and bool(need[4]), c_0 is not None and bool(need[5]),
                 *map(bool, need[6:]))
        lstm = ctx.cfg.mode == _lib.LSTM
        dx, dh_0, dc_0, *dws = _Backward.apply(ctx.cfg, needs, x_tm, y, reserve, h_0, c_0, dy, dh_n,
                                               dc_n if lstm else None, *weights)
        keep = lambda g, n: g if n else None  # noqa: E731
        return (keep(dx, needs[0]), None, None, None, keep(dh_0, needs[1]), keep(dc_0, needs[2]),
                *(keep(g, n) for g, n in zip(dws, needs[3:])))

    @staticmethod
    def jvp(ctx, x_dot, _cfg, _rng, _save, h0_dot, c0_dot, *w_dots):
        x_tm, y, reserve, h_0, c_0, *weights = ctx.saved_tensors
        y_dot, h_n_dot, c_n_dot = tangent(ctx.cfg, x_tm, y, reserve, h_0, c_0, x_dot, h0_dot, c0_dot, weights, w_dots)
        return y_dot, h_n_dot, c_n_dot if c_n_dot is not None else None, None

    @staticmethod
    def vmap(info, in_dims, x_tm, cfg, rng_state, save, h_0, c_0, *weights):
        M = info.batch_size
        if cfg.models > 1:
            raise _lib.B200RNNError("b200rnn: nested vmap over a recurrent module is not supported")
        x_dim, _, rng_dim, _, h_dim, c_dim, *w_dims = in_dims
        rng_stride = 0
        if cfg.training and cfg.dropout > 0 and cfg.num_layers > 1:
            if info.randomness == "error":
                raise RuntimeError(_RANDOMNESS_ERROR)
            if rng_state is not None and rng_dim is not None:
                if info.randomness == "same":
                    raise _lib.B200RNNError("b200rnn: vmap(randomness='same') draws one dropout mask for every model "
                                            "from one _rng_state; got a batched one")
                rng_state = rng_state.movedim(rng_dim, 0)
                if not rng_state.is_contiguous():   # the kernels advance each row in place
                    raise _lib.B200RNNError("b200rnn: a batched _rng_state must be a contiguous [M, 2] block")
                rng_stride = rng_state.stride(0)
            elif info.randomness == "different":
                rng_stride = -1
        elif rng_state is not None and rng_dim is not None:
            rng_state = rng_state.movedim(rng_dim, 0)
            rng_stride = rng_state.stride(0)
        cfg_m = dataclasses.replace(cfg, models=M, rng_stride=rng_stride)
        # the caller decided `save` on the batched tensors, whose requires_grad says nothing of autograd outside vmap
        save = save or (torch.is_grad_enabled() and any(t is not None and t.requires_grad
                                                         for t in (x_tm, h_0, c_0, *weights)))
        x_m = _to_models(x_tm, x_dim, M, dense=False)
        if x_m.stride(-1) != 1 and x_m.size(-1) != 1:
            x_m = x_m.contiguous()
        w_m = [_weight_models(w, d, M) for w, d in zip(weights, w_dims)]
        if M == 1:
            cfg_m = cfg
            rng_state = _one_model([rng_state], M)[0] if rng_stride > 0 else rng_state
        h_m, c_m = _to_models(h_0, h_dim, M, True), _to_models(c_0, c_dim, M, True)
        x_m, h_m, c_m, *w_m = _one_model([x_m, h_m, c_m, *w_m], M)
        out_dims = (0, 0, 0 if cfg.mode == _lib.LSTM else None, 0)
        out = _Forward.apply(x_m, cfg_m, rng_state, save, h_m, c_m, *w_m)
        return _with_model_dim(out, out_dims, M), out_dims


class _Backward(torch.autograd.Function):
    """``(dx, dh_0, dc_0, *weight grads)`` of :class:`_Forward`; ``needs`` = [dx, dh_0, dc_0, one per weight], an
    empty stand-in for what is not needed. Not differentiable again."""

    @staticmethod
    def forward(cfg, needs, x_tm, y, reserve, h_0, c_0, dy, dh_n, dc_n, *weights):
        dx, dh_0, dc_0, dws = F._rnn_backward_impl(cfg, x_tm, y, reserve, h_0, c_0, weights, dy, dh_n, dc_n, None,
                                                   needs[0], needs[1], needs[2], needs[3:], None, separate=True)
        none = lambda g: g if g is not None else x_tm.new_empty(0)  # noqa: E731
        return (none(dx), none(dh_0), none(dc_0), *map(none, dws))

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    def backward(ctx, *grads):
        raise _lib.B200RNNError("b200rnn: the recurrence's backward is not differentiable (no double backward)")

    @staticmethod
    def jvp(ctx, *tangents):
        raise _lib.B200RNNError("b200rnn: forward-over-reverse (hessian, jvp of grad) is not supported: the "
                                "recurrence's backward has no forward-mode derivative")

    @staticmethod
    def vmap(info, in_dims, cfg, needs, x_tm, y, reserve, h_0, c_0, dy, dh_n, dc_n, *weights):
        M = info.batch_size
        if cfg.models > 1:
            raise _lib.B200RNNError("b200rnn: nested vmap over a recurrent module is not supported")
        _, _, x_dim, y_dim, r_dim, h_dim, c_dim, dy_dim, dhn_dim, dcn_dim, *w_dims = in_dims
        # still wrapped below this vmap: a jvp (hessian = jacfwd(jacrev)) differentiates the backward in forward mode
        if any(torch._C._functorch.is_functorch_wrapped_tensor(t) for t in (x_tm, y, dy, *weights) if t is not None):
            raise _lib.B200RNNError("b200rnn: forward-over-reverse (hessian, jvp of grad) is not supported: the "
                                    "recurrence's backward has no forward-mode derivative")
        cfg_m = dataclasses.replace(cfg, models=M) if M > 1 else cfg
        x_m = _to_models(x_tm, x_dim, M, dense=False)
        if x_m.stride(-1) != 1 and x_m.size(-1) != 1:
            x_m = x_m.contiguous()
        dense = lambda t, d: _to_models(t, d, M, True)  # noqa: E731
        w_m = [_weight_models(w, d, M) for w, d in zip(weights, w_dims)]
        args = _one_model([x_m, dense(y, y_dim), dense(reserve, r_dim), dense(h_0, h_dim), dense(c_0, c_dim),
                           dense(dy, dy_dim), dense(dh_n, dhn_dim), dense(dc_n, dcn_dim), *w_m], M)
        out = _Backward.forward(cfg_m, needs, *args)
        wanted = (needs[0], needs[1] and h_0 is not None, needs[2] and c_0 is not None, *needs[3:])
        out_dims = tuple(0 if n else None for n in wanted)
        return _with_model_dim(out, out_dims, M), out_dims


class _Tangent(torch.autograd.Function):
    """``(y', h_n', c_n')`` of :class:`_Forward` (``c_n'`` an empty stand-in but for the LSTM) from the primal's
    ``x_tm``, ``y``, ``reserve`` and states and the tangents of ``x_tm``, ``h_0``, ``c_0`` and each weight (None = 0;
    ``weights_and_dots`` is the weights, then one tangent per weight). Not differentiable."""

    @staticmethod
    def forward(cfg, x_tm, y, reserve, h_0, c_0, x_dot, h0_dot, c0_dot, *weights_and_dots):
        n = len(weights_and_dots) // 2
        y_dot, h_n_dot, c_n_dot = F._rnn_tangent_impl(cfg, x_tm, y, reserve, h_0, c_0, weights_and_dots[:n], x_dot,
                                                      h0_dot, c0_dot, weights_and_dots[n:])
        return y_dot, h_n_dot, c_n_dot if c_n_dot is not None else y_dot.new_empty(0)

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    def backward(ctx, *grads):
        raise _lib.B200RNNError("b200rnn: reverse-over-forward (the gradient of a jvp tangent) is not supported")

    @staticmethod
    def vmap(info, in_dims, cfg, x_tm, y, reserve, h_0, c_0, x_dot, h0_dot, c0_dot, *weights_and_dots):
        """M tangent directions over one primal (``jacfwd``): one library call, each tangent a dense [M, ...] block"""
        M = info.batch_size
        n = len(weights_and_dots) // 2
        _, x_dim, y_dim, r_dim, h_dim, c_dim, xd_dim, hd_dim, cd_dim, *wd = in_dims
        if any(d is not None for d in (x_dim, y_dim, r_dim, h_dim, c_dim, *wd[:n])):
            raise _lib.B200RNNError("b200rnn: forward-mode AD over a vmap-batched primal (a jvp inside vmap over "
                                    "models or samples) is not supported; vmap over the tangents only (jacfwd)")
        dense = lambda t, d: _to_models(t, d, M, True)  # noqa: E731
        dots = [dense(t, d) for t, d in zip(weights_and_dots[n:], wd[n:])]
        y_dot, h_n_dot, c_n_dot = F._rnn_tangent_impl(cfg, x_tm, y, reserve, h_0, c_0, weights_and_dots[:n],
                                                      dense(x_dot, xd_dim), dense(h0_dot, hd_dim),
                                                      dense(c0_dot, cd_dim), dots, directions=M)
        lstm = cfg.mode == _lib.LSTM
        out = (y_dot, h_n_dot, c_n_dot if lstm else y_dot.new_empty(0))
        out_dims = (0, 0, 0 if lstm else None)
        return _with_model_dim(out, out_dims, M), out_dims


def tangent(cfg: F.RNNConfig, x_tm, y, reserve, h_0, c_0, x_dot, h0_dot, c0_dot, weights, w_dots):
    """``(y', h_n', c_n')`` through :class:`_Tangent`, ``c_n'`` None but for the LSTM"""
    y_dot, h_n_dot, c_n_dot = _Tangent.apply(cfg, x_tm, y, reserve, h_0, c_0, x_dot, h0_dot, c0_dot, *weights,
                                             *w_dots)
    return y_dot, h_n_dot, c_n_dot if cfg.mode == _lib.LSTM else None


def rnn_forward(x_tm: torch.Tensor, cfg: F.RNNConfig, rng_state: Optional[torch.Tensor], save: bool,
                h_0: Optional[torch.Tensor], c_0: Optional[torch.Tensor], weights: Sequence[torch.Tensor]):
    """``functional.rnn_forward`` under a functorch transform, after its argument checks: ``(y, h_n)``, or
    ``(y, h_n, c_n)`` for the LSTM"""
    y, h_n, c_n, _ = _Forward.apply(x_tm, cfg, rng_state, bool(save), h_0, c_0, *weights)
    return (y, h_n, c_n) if cfg.mode == _lib.LSTM else (y, h_n)
