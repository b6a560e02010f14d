"""Stacked GRU / LSTM / RNN as a chain of stock one-layer modules, with optional inter-layer dropout masks.

A stock ``nn.GRU`` / ``nn.LSTM`` / ``nn.RNN(num_layers=L)`` feeds layer l the output of layer l - 1, dropped in train
mode. Here the same stack is L one-layer stock modules (``split_layers``) run one after another (``chained``), so that
the dropout between them can be given as fixed masks: ``masks[l]`` multiplies layer l's output (the factors of
``oracle.philox.dropout_factor``: 1 / (1 - p) or 0), which is what the library's ``dropout_kernel`` draws. In float64
the chain is the float64 reference of a stacked call; in fp32 it is stock torch's own fp32 evaluation of it.
"""
from __future__ import annotations

import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

PARAMS = ("weight_ih", "weight_hh", "bias_ih", "bias_hh", "weight_hr")


def _one_layer_like(ref: torch.nn.RNNBase, input_size: int) -> torch.nn.RNNBase:
    kw = dict(bidirectional=ref.bidirectional, batch_first=False)
    if isinstance(ref, torch.nn.LSTM):
        return torch.nn.LSTM(input_size, ref.hidden_size, proj_size=ref.proj_size, **kw)
    if isinstance(ref, torch.nn.GRU):
        return torch.nn.GRU(input_size, ref.hidden_size, **kw)
    return torch.nn.RNN(input_size, ref.hidden_size, nonlinearity=ref.nonlinearity, **kw)


def split_layers(ref: torch.nn.RNNBase) -> list:
    """L one-layer stock modules holding layer l's parameters of ``ref`` (same dtype and device), time-major"""
    D = 2 if ref.bidirectional else 1
    width = D * (ref.proj_size or ref.hidden_size)
    layers = []
    for l in range(ref.num_layers):
        m = _one_layer_like(ref, ref.input_size if l == 0 else width)
        m = m.to(dtype=next(ref.parameters()).dtype, device=next(ref.parameters()).device)
        with torch.no_grad():
            for name, p in m.named_parameters():
                p.copy_(getattr(ref, name.replace("_l0", f"_l{l}")))
        layers.append(m)
    return layers


def chained(layers: list, x: torch.Tensor, lengths=None, hx=None, masks=None):
    """Run ``layers`` (one-layer stock modules) one after another on time-major ``x`` [T, B, I].

    ``lengths``: per-row lengths (a ragged batch, through ``PackedSequence``; the padding of y is 0). ``hx``: None, h_0
    or (h_0, c_0), each [L * D, B, *] as the stacked module takes it. ``masks``: None, or L - 1 factors (tensors
    broadcasting against [T, B, D * HO]) that multiply each inner layer's output. Differentiable in x, hx and every
    layer's parameters. Returns (y, states): states is (h_n,) or (h_n, c_n), each [L * D, B, *]."""
    T = x.shape[0]
    D = 2 if layers[0].bidirectional else 1
    states_in = None if hx is None else (tuple(hx) if isinstance(hx, (tuple, list)) else (hx,))
    h, finals = x, []
    for l, m in enumerate(layers):
        st = None if states_in is None else tuple(s[l * D:(l + 1) * D] for s in states_in)
        st = None if st is None else (st if len(st) == 2 else st[0])
        inp = h if lengths is None else pack_padded_sequence(h, lengths, enforce_sorted=False)
        out, s = m(inp, st)
        h = out if lengths is None else pad_packed_sequence(out, total_length=T)[0]
        finals.append(s if isinstance(s, tuple) else (s,))
        if masks is not None and l + 1 < len(layers):
            h = h * masks[l]
    states = tuple(torch.cat([f[i] for f in finals]) for i in range(len(finals[0])))
    return h, states
