"""Autograd bridge between PyTorch tensors and the C-ABI library.

``rnn_forward`` is what ``b200rnn.GRU.forward`` / ``b200rnn.LSTM.forward`` call in place of ``_VF.gru`` /
``_VF.lstm`` (torch/nn/modules/rnn.py:1449 / :1169). PyTorch is only plumbing here: it owns the device
memory (``torch.empty`` -> caching allocator, CUDA-graph friendly) and the current stream; all arithmetic
happens in ``lib/libb200rnn.so``. CPU tensors are rejected — there is no fallback path.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Optional, Sequence

import torch

from . import _lib


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


def _require_cuda_f32(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise _lib.B200RNNError(
            f"b200rnn: {name} is on {t.device}; this library runs on CUDA (sm_90a) only and has no CPU path"
        )
    if t.dtype != torch.float32:
        raise _lib.B200RNNError(f"b200rnn: {name} must be float32 (got {t.dtype})")


def _tm_view(x: torch.Tensor) -> torch.Tensor:
    """Return a logical [T,B,F] tensor whose feature stride is 1 (copy only if it is not)."""
    if x.stride(2) != 1 and x.size(2) != 1:
        x = x.contiguous()
    return x


def _make_desc(cfg: RNNConfig, B: int, T: int, save: bool, accumulate: bool = False,
               fused_ln: bool = False) -> _lib.Desc:
    flags = 0
    if save:
        flags |= _lib.FLAG_SAVE_FOR_BACKWARD
    if accumulate:
        flags |= _lib.FLAG_ACCUMULATE_GRADS
    if fused_ln:
        flags |= _lib.FLAG_FUSED_LN
    return _lib.Desc(cfg.mode, B, T, cfg.input_size, cfg.hidden_size, cfg.num_layers, cfg.num_dirs,
                     1 if cfg.training else 0, float(cfg.dropout), flags)


def _stream_ptr(device=None) -> int:
    """Raw handle of the current stream OF ``device`` (not of the process-wide current device)."""
    return torch.cuda.current_stream(device).cuda_stream


def _on(device):
    """Make ``device`` current around a library call: the C side queries / configures the CURRENT device
    (``cudaFuncSetAttribute``, occupancy, SM count), and stock nn.GRU / nn.LSTM work on whatever device their tensors
    live on, so the drop-in has to as well (module on cuda:1 while cuda:0 is the process default)."""
    return torch.cuda.device(device)


class _RNNFunction(torch.autograd.Function):
    """y, h_n[, c_n] = RNN(x, weights); x is the logical time-major view [T,B,I]."""

    @staticmethod
    def forward(ctx, x_tm: torch.Tensor, cfg: RNNConfig, rng_state: Optional[torch.Tensor], grad_sink,
                lengths: Optional[torch.Tensor], save: bool, *weights: torch.Tensor):
        lib = _lib.load()
        T, B, _ = x_tm.shape
        H, L, D = cfg.hidden_size, cfg.num_layers, cfg.num_dirs
        dev = x_tm.device
        # `save` is decided by the caller: grad mode is always off in here, and needs_input_grad is True for
        # requires_grad weights even under torch.no_grad() (it would allocate the reserve and store gates for nothing)
        save = bool(save) and any(ctx.needs_input_grad)
        desc = _make_desc(cfg, B, T, save)
        rbytes, sbytes = _lib.workspace_bytes(desc)
        reserve = torch.empty(rbytes if save else 0, dtype=torch.uint8, device=dev)
        scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
        if cfg.batch_first:
            y = torch.empty(B, T, D * H, dtype=torch.float32, device=dev)
            ys_t, ys_b = D * H, T * D * H
        else:
            y = torch.empty(T, B, D * H, dtype=torch.float32, device=dev)
            ys_t, ys_b = B * D * H, D * H
        h_n = torch.empty(L * D, B, H, dtype=torch.float32, device=dev)
        c_n = torch.empty(L * D, B, H, dtype=torch.float32, device=dev) if cfg.mode == _lib.LSTM else None
        params = _lib.ptr_array([w.data_ptr() for w in weights])
        if B > 0 and T > 0:
            with _on(dev):
                rc = lib.b200rnn_forward_fused(
                    ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params,
                    y.data_ptr(), ys_t, ys_b, h_n.data_ptr(), c_n.data_ptr() if c_n is not None else None,
                    reserve.data_ptr() if save else None, scratch.data_ptr(),
                    0, 0, rng_state.data_ptr() if rng_state is not None else None, None, None, 0.0, None,
                    lengths.data_ptr() if lengths is not None else None, None, _stream_ptr(dev))
            _lib.check(rc, "b200rnn_forward")
        else:
            h_n.zero_()
            if c_n is not None:
                c_n.zero_()
        if save:
            ctx.cfg = cfg
            ctx.grad_sink = grad_sink
            ctx.ys = (ys_t, ys_b)
            ctx.lengths = lengths
            ctx.save_for_backward(x_tm, y, reserve, *weights)
        if c_n is None:
            return y, h_n
        return y, h_n, c_n

    @staticmethod
    def backward(ctx, dy, dh_n, dc_n=None):
        lib = _lib.load()
        cfg: RNNConfig = ctx.cfg
        x_tm, y, reserve, *weights = ctx.saved_tensors
        T, B, _ = x_tm.shape
        H, L, D = cfg.hidden_size, cfg.num_layers, cfg.num_dirs
        dev = x_tm.device
        ys_t, ys_b = ctx.ys

        if dy is None:
            dy = torch.zeros_like(y)
        if dy.stride(2) != 1 and dy.size(2) != 1:
            dy = dy.contiguous()
        if cfg.batch_first:
            dys_t, dys_b = dy.stride(1), dy.stride(0)
        else:
            dys_t, dys_b = dy.stride(0), dy.stride(1)
        if dh_n is not None:
            dh_n = dh_n.contiguous()
        if dc_n is not None:
            dc_n = dc_n.contiguous()

        need_dx = ctx.needs_input_grad[0]
        dx = torch.empty_like(x_tm) if need_dx else None
        if dx is not None and dx.stride(2) != 1 and dx.size(2) != 1:
            dx = torch.empty(x_tm.shape, dtype=torch.float32, device=dev)

        # weight gradients: either straight into caller-provided views (a flat all-reduce bucket) or into one
        # fresh flat buffer that is returned to autograd as views
        sink = ctx.grad_sink
        w_needed = [ctx.needs_input_grad[6 + i] for i in range(len(weights))]
        grads_out: list = [None] * len(weights)
        accumulate = False
        if sink is not None:
            targets = sink(weights)  # list of tensors (same shapes) or None entries
            accumulate = True
            dptrs = [t.data_ptr() if (t is not None and n) else None for t, n in zip(targets, w_needed)]
        else:
            sizes = [w.numel() if n else 0 for w, n in zip(weights, w_needed)]
            flat = torch.empty(sum(sizes), dtype=torch.float32, device=dev)
            dptrs, off = [], 0
            for i, (w, n) in enumerate(zip(weights, w_needed)):
                if n:
                    g = flat[off:off + w.numel()].view_as(w)
                    off += w.numel()
                    grads_out[i] = g
                    dptrs.append(g.data_ptr())
                else:
                    dptrs.append(None)

        desc = _make_desc(cfg, B, T, True, accumulate)
        _, sbytes = _lib.workspace_bytes(desc)
        scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
        params = _lib.ptr_array([w.data_ptr() for w in weights])
        dparams = _lib.ptr_array(dptrs)
        if B > 0 and T > 0:
            with _on(dev):
                rc = lib.b200rnn_backward(
                    ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params,
                    y.data_ptr(), ys_t, ys_b, dy.data_ptr(), dys_t, dys_b,
                    dh_n.data_ptr() if dh_n is not None else None,
                    dc_n.data_ptr() if dc_n is not None else None,
                    reserve.data_ptr(), scratch.data_ptr(),
                    dx.data_ptr() if dx is not None else None,
                    dx.stride(0) if dx is not None else 0, dx.stride(1) if dx is not None else 0,
                    dparams, ctx.lengths.data_ptr() if ctx.lengths is not None else None, _stream_ptr(dev))
            _lib.check(rc, "b200rnn_backward")
        else:
            for g in grads_out:
                if g is not None:
                    g.zero_()
        return (dx, None, None, None, None, None, *grads_out)


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
                pooled.data_ptr(), None, None, _stream_ptr(dev))
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
        sink = ctx.grad_sink
        w_needed = [ctx.needs_input_grad[7 + i] for i in range(len(weights))]
        grads_out: list = [None] * len(weights)
        accumulate = False
        if sink is not None:
            targets = sink(weights)
            accumulate = True
            dptrs = [t.data_ptr() if (t is not None and n) else None for t, n in zip(targets, w_needed)]
        else:
            sizes = [(w.numel() + 63) // 64 * 64 if n else 0 for w, n in zip(weights, w_needed)]
            flat = torch.empty(sum(sizes), dtype=torch.float32, device=dev)
            dptrs, off = [], 0
            for i, (w, n) in enumerate(zip(weights, w_needed)):
                if n:
                    g = flat[off:off + w.numel()].view_as(w)
                    off += sizes[i]
                    grads_out[i] = g
                    dptrs.append(g.data_ptr())
                else:
                    dptrs.append(None)
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
    x_tm = _tm_view(x.transpose(0, 1) if cfg.batch_first else x)
    return _LNRNNPoolFunction.apply(x_tm, cfg, rng_state, grad_sink, ln_weight, ln_bias, ln_eps, *weights)


def rnn_forward(x: torch.Tensor, weights: Sequence[torch.Tensor], cfg: RNNConfig,
                rng_state: Optional[torch.Tensor] = None, grad_sink=None, lengths: Optional[torch.Tensor] = None):
    """Run the multi-layer GRU/LSTM. ``x`` is [T,B,I] (or [B,T,I] if ``cfg.batch_first``), any strides.

    Returns ``(y, h_n)`` for GRU and ``(y, h_n, c_n)`` for LSTM, laid out like torch.nn.GRU/LSTM outputs.
    """
    _require_cuda_f32(x, "input")
    if x.dim() != 3:
        raise NotImplementedError("b200rnn: only batched 3-D input is supported (the reference never uses 2-D)")
    for i, w in enumerate(weights):
        _require_cuda_f32(w, f"weight[{i}]")
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
    save = torch.is_grad_enabled() and (x.requires_grad or any(w.requires_grad for w in weights))
    return _RNNFunction.apply(x_tm, cfg, rng_state, grad_sink, lengths, save, *weights)


@torch.no_grad()
def rnn_forward_fused(x: torch.Tensor, weights: Sequence[torch.Tensor], cfg: RNNConfig,
                      rng_state: Optional[torch.Tensor] = None, ln_weight: Optional[torch.Tensor] = None,
                      ln_bias: Optional[torch.Tensor] = None, ln_eps: float = 1e-5, pool_sum: bool = False,
                      wcache: Optional[torch.Tensor] = None):
    """No-grad forward with the shell fusions of ``b200rnn_forward_fused``: optional LayerNorm prologue on ``x``
    and, with ``pool_sum``, the sum over time of the output instead of the sequence (``[B, D*H]``).

    Mirrors ``x = ln(x); x, _ = gru(x); x = x.sum(dim=1)`` (fuse_net_whole.py:360-362). Returns ``(out, h_n[, c_n])``.
    """
    lib = _lib.load()
    _require_cuda_f32(x, "input")
    x_tm = _tm_view(x.transpose(0, 1) if cfg.batch_first else x)
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
    with _on(dev):
        rc = lib.b200rnn_forward_fused(
            ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params, y_ptr, ys_t, ys_b,
            h_n.data_ptr(), c_n.data_ptr() if c_n is not None else None, None, scratch.data_ptr(), 0, 0,
            rng_state.data_ptr() if rng_state is not None else None,
            ln_weight.data_ptr() if ln_weight is not None else None,
            ln_bias.data_ptr() if ln_bias is not None else None,
            float(ln_eps), pool_ptr, None, wcache.data_ptr() if wcache is not None else None, _stream_ptr(dev))
    _lib.check(rc, "b200rnn_forward_fused")
    return (out, h_n) if c_n is None else (out, h_n, c_n)


def prepare_weights(weights: Sequence[torch.Tensor], cfg: RNNConfig) -> torch.Tensor:
    """TF32 hi/lo split of every ``weight_ih`` (``b200rnn_prepare_weights``): the weight cache ``rnn_forward_fused``
    accepts so that frozen encoders split their weights once instead of once per step."""
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
