"""ORACLE — test infrastructure only (never imported by the product path).

Emulation of b200rnn's single-pass TF32 mode (``B200RNN_FLAG_TF32``, on while torch's fp32 matmul precision is
``"tf32"``) in float64. The kernels round some operands to TF32 and multiply them once; everything else stays fp32.
This restatement rounds exactly those operands and computes the rest in float64:

  forward   the input projection x_l W_ih^T: x_l (layer 0: x or LayerNorm(x); layer l > 0: the, possibly dropped, output
            of layer l-1) and W_ih;
            the recurrent product W_hh h_{t-1} only in the GRU-256 tensor-core config tc8 (``rec_round=True``): W_hh and
            the exchanged h_{t-1}. The cell update itself keeps the unrounded h_{t-1};
  backward  the operands of the three GEMMs: dW_ih = dG^T x_l, dW_hh = dGh^T h_prev and dx_l = dG W_ih. The BPTT
            recurrence (dh = ... + dGh W_hh) and the bias sums stay unrounded.

Teacher forcing (``observed``): a rounded operand is a step function of its fp32 input, so an emulation that carries
its own float64 state rounds some values to the other TF32 neighbour than the kernels did, and each such value moves a
product by a TF32 ulp (~1e-5 on the outputs after a few hundred steps). Given the outputs the kernels produced, layer
by layer, the emulation instead takes layer l's input from layer l-1's observed output and h_{t-1} from this layer's
observed output, so it rounds the very values the kernels rounded and each step is compared on its own.

The GEMMs run on the tensor cores for layer widths that are multiples of 128 (backward) / 32 (forward); the tests use
such shapes, so every GEMM operand is rounded here. With ``rounding=False`` the arithmetic is operation for operation
that of oracle/rnn_numpy.py (tests/test_tf32_mode_cpu.py checks that they agree exactly). Inter-layer dropout is not
modelled, as in rnn_numpy.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .rnn_numpy import _gates, _sigmoid


def round_tf32(x) -> np.ndarray:
    """Round to TF32 as ``cvt.rna.tf32.f32`` does: x is taken as float32, its 13 low mantissa bits are rounded away to
    nearest with ties away from zero (10 mantissa bits remain). Returns float32."""
    a = np.ascontiguousarray(np.asarray(x, dtype=np.float32))
    bits = a.view(np.uint32)
    # sign-magnitude: adding half of the dropped range to the magnitude bits rounds |x| half-up, i.e. ties away from 0
    out = ((bits + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).astype(np.uint32)
    return out.view(np.float32).reshape(a.shape)


def _identity(x):
    return x


def _layer_forward(mode, x, w_ih, w_hh, b_ih, b_hh, reverse, lengths, R, rec_round, h_obs=None):
    """rnn_numpy._layer_forward with the rounded operands: R(x) R(W_ih)^T, and R(h) R(W_hh)^T when rec_round.
    h_obs [T,B,H]: the observed output of this direction; a live step starts from its previous observed output (0
    before the first step, which is also what a padded output row holds)."""
    T, B, _ = x.shape
    live = None if lengths is None else (np.arange(T)[:, None] < np.asarray(lengths)[None, :])
    H = w_hh.shape[1]
    Rh = R if rec_round else _identity
    xr, wir, whr = R(x), R(w_ih), Rh(w_hh)
    h = np.zeros((B, H), dtype=x.dtype)
    c = np.zeros((B, H), dtype=x.dtype)
    y = np.zeros((T, B, H), dtype=x.dtype)
    cache: List[dict] = [None] * T  # type: ignore
    order = range(T - 1, -1, -1) if reverse else range(T)
    for t in order:
        if h_obs is not None:
            tp = t + 1 if reverse else t - 1
            h_prev = h_obs[tp] if 0 <= tp < T else np.zeros_like(h)
            h = h_prev if live is None else np.where(live[t][:, None], h_prev, h)
        gi = xr[t] @ wir.T + b_ih
        gh = Rh(h) @ whr.T + b_hh
        if mode == "gru":
            r = _sigmoid(gi[:, :H] + gh[:, :H])
            z = _sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
            hn = gh[:, 2 * H:]
            n = np.tanh(gi[:, 2 * H:] + r * hn)
            h_new = (1.0 - z) * n + z * h
            cache[t] = dict(r=r, z=z, n=n, hn=hn, h_prev=h)
        else:
            a = gi + gh
            i = _sigmoid(a[:, :H])
            f = _sigmoid(a[:, H:2 * H])
            g = np.tanh(a[:, 2 * H:3 * H])
            o = _sigmoid(a[:, 3 * H:])
            c_new = f * c + i * g
            h_new = o * np.tanh(c_new)
            cache[t] = dict(i=i, f=f, g=g, o=o, c=c_new, c_prev=c, h_prev=h)
            if live is not None:
                c_new = np.where(live[t][:, None], c_new, c)
            c = c_new
        if live is not None:
            y[t] = np.where(live[t][:, None], h_new, 0.0)
            h = np.where(live[t][:, None], h_new, h)
        else:
            h = h_new
            y[t] = h
    return y, h, c, cache


def _layer_backward(mode, x, w_ih, w_hh, cache, dy, dh_last, dc_last, reverse, lengths, R):
    """rnn_numpy._layer_backward with the GEMM operands rounded: R(dG) R(W_ih), R(dG)^T R(x), R(dGh)^T R(h_prev)."""
    T, B, _ = x.shape
    live = None if lengths is None else (np.arange(T)[:, None] < np.asarray(lengths)[None, :])
    H = w_hh.shape[1]
    xr, wir = R(x), R(w_ih)
    dx = np.zeros_like(x)
    dw_ih = np.zeros_like(w_ih)
    dw_hh = np.zeros_like(w_hh)
    db_ih = np.zeros(w_ih.shape[0], dtype=x.dtype)
    db_hh = np.zeros(w_ih.shape[0], dtype=x.dtype)
    dh = dh_last.copy()
    dc = dc_last.copy()
    order = range(T) if reverse else range(T - 1, -1, -1)
    for t in order:
        k = cache[t]
        m = None if live is None else live[t][:, None]
        dht = dh + (dy[t] if m is None else np.where(m, dy[t], 0.0))
        if mode == "gru":
            r, z, n, hn, h_prev = k["r"], k["z"], k["n"], k["hn"], k["h_prev"]
            dn = dht * (1.0 - z) * (1.0 - n * n)
            dz = dht * (h_prev - n) * z * (1.0 - z)
            dr = dn * hn * r * (1.0 - r)
            dgi = np.concatenate([dr, dz, dn], axis=1)
            dgh = np.concatenate([dr, dz, dn * r], axis=1)
            if m is not None:
                dgi, dgh = dgi * m, dgh * m
                dh = np.where(m, dht * z, dht) + dgh @ w_hh
            else:
                dh = dht * z + dgh @ w_hh
        else:
            i, f, g, o, c, c_prev, h_prev = k["i"], k["f"], k["g"], k["o"], k["c"], k["c_prev"], k["h_prev"]
            tc = np.tanh(c)
            do = dht * tc * o * (1.0 - o)
            dct = dc + dht * o * (1.0 - tc * tc)
            di = dct * g * i * (1.0 - i)
            df = dct * c_prev * f * (1.0 - f)
            dg = dct * i * (1.0 - g * g)
            dgi = np.concatenate([di, df, dg, do], axis=1)
            if m is not None:
                dgi = dgi * m
                dc = np.where(m, dct * f, dc)
                dh = np.where(m, 0.0, dht) + dgi @ w_hh
            else:
                dc = dct * f
                dh = dgi @ w_hh
            dgh = dgi
        dgir = R(dgi)
        dx[t] = dgir @ wir
        dw_ih += dgir.T @ xr[t]
        dw_hh += R(dgh).T @ R(h_prev)
        db_ih += dgi.sum(axis=0)
        db_hh += dgh.sum(axis=0)
    return dx, dw_ih, dw_hh, db_ih, db_hh


class Tf32RNN:
    """Multi-layer (bi)directional GRU/LSTM, time-major [T,B,*], as b200rnn computes it in single-pass TF32 mode.

    ``rec_round``: the recurrence is the GRU-256 tensor-core config tc8 (its W_hh h_{t-1} is rounded too); every other
    recurrence config is fp32 FFMA. ``rounding=False`` turns every rounding off (then this is rnn_numpy.NumpyRNN)."""

    def __init__(self, mode: str, weights: Sequence[np.ndarray], num_layers: int, bidirectional: bool,
                 rec_round: bool = False, rounding: bool = True):
        _gates(mode)
        self.mode = mode
        self.L = num_layers
        self.D = 2 if bidirectional else 1
        assert len(weights) == 4 * self.L * self.D
        self.w = [np.asarray(w, dtype=np.float64) for w in weights]
        self.R = (lambda a: round_tf32(a).astype(np.float64)) if rounding else _identity
        self.rec_round = rec_round
        self._saved = None

    def _p(self, l: int, d: int):
        base = 4 * (l * self.D + d)
        return self.w[base:base + 4]

    def forward(self, x: np.ndarray, lengths=None, observed: Optional[Sequence[np.ndarray]] = None):
        """x [T,B,I]; ``observed``: the kernels' output of every layer ([T,B,D*H] each) for teacher forcing."""
        x = np.asarray(x, dtype=np.float64)
        self._lengths = None if lengths is None else np.asarray(lengths, dtype=np.int64)
        inp = x
        h_n, c_n, saved = [], [], []
        for l in range(self.L):
            outs, caches = [], []
            if observed is not None and l > 0:
                inp = np.asarray(observed[l - 1], dtype=np.float64)
            for d in range(self.D):
                w_ih, w_hh, b_ih, b_hh = self._p(l, d)
                H = w_hh.shape[1]
                h_obs = None if observed is None else np.asarray(observed[l], np.float64)[:, :, d * H:(d + 1) * H]
                y, h, c, cache = _layer_forward(self.mode, inp, w_ih, w_hh, b_ih, b_hh, d == 1, self._lengths, self.R,
                                                self.rec_round, h_obs)
                outs.append(y)
                caches.append(cache)
                h_n.append(h)
                c_n.append(c)
            saved.append((inp, caches))
            inp = np.concatenate(outs, axis=2) if self.D == 2 else outs[0]
        self._saved = saved
        h_n = np.stack(h_n)
        if self.mode == "lstm":
            return inp, h_n, np.stack(c_n)
        return inp, h_n

    def backward(self, dy: np.ndarray, dh_n: Optional[np.ndarray] = None, dc_n: Optional[np.ndarray] = None):
        """Returns (dx, [dparams in nn order])."""
        assert self._saved is not None, "call forward first"
        dy = np.asarray(dy, dtype=np.float64)
        grads: Dict[Tuple[int, int], tuple] = {}
        for l in range(self.L - 1, -1, -1):
            inp, caches = self._saved[l]
            T, B, _ = inp.shape
            H = self._p(l, 0)[1].shape[1]
            dinp = np.zeros_like(inp)
            for d in range(self.D):
                w_ih, w_hh, _, _ = self._p(l, d)
                idx = l * self.D + d
                dh_last = np.zeros((B, H)) if dh_n is None else np.asarray(dh_n[idx], np.float64)
                dc_last = np.zeros((B, H)) if dc_n is None else np.asarray(dc_n[idx], np.float64)
                dyd = dy[:, :, d * H:(d + 1) * H]
                dx, dw_ih, dw_hh, db_ih, db_hh = _layer_backward(self.mode, inp, w_ih, w_hh, caches[d], dyd, dh_last,
                                                                 dc_last, d == 1, self._lengths, self.R)
                dinp += dx
                grads[(l, d)] = (dw_ih, dw_hh, db_ih, db_hh)
            dy = dinp
        flat = []
        for l in range(self.L):
            for d in range(self.D):
                flat.extend(grads[(l, d)])
        return dy, flat
