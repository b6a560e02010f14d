"""ORACLE — test infrastructure only (never imported by the product path).

A numpy restatement, in float64 by default, of the multi-layer GRU / bidirectional LSTM the reference reaches
through ``torch.nn.GRU`` / ``torch.nn.LSTM`` (call sites audio_gru_whole.py:59-60,105; text_bilstm_whole.py:54-56,105;
fuse_net_whole.py:266-268,281-286,347,361). The arithmetic itself lives in a third-party dependency that is not part
of the reference — PyTorch (the reference pins no version; the oracle version is the installed torch 2.11.0) — so this
file restates the published equations:

  GRU  (torch/nn/modules/rnn.py:1221-1224), gate order r,z,n:
      r = s(W_ir x + b_ir + W_hr h + b_hr);  z = s(W_iz x + b_iz + W_hz h + b_hz)
      n = tanh(W_in x + b_in + r * (W_hn h + b_hn));  h' = (1 - z) * n + z * h
  LSTM (rnn.py:842-847), gate order i,f,g,o:
      i,f,o = s(.), g = tanh(.);  c' = f * c + i * g;  h' = o * tanh(c')
  parameters per layer / direction weight_ih[G*H, I_l], weight_hh[G*H, H], bias_ih, bias_hh (rnn.py:171-216);
  h0 = c0 = 0 (rnn.py:1432-1440); the reverse direction scans t = T-1..0; layer l>0 consumes concat(fwd, rev);
  h_n / c_n are ordered (l0 fwd, l0 rev, l1 fwd, ...).

Parity pinning: the reference repository has no tests or golden vectors for this path (SURVEY.md §8c, "parity
unpinned" by the reference itself); this restatement is pinned instead against the executed dependency
(tests/test_oracle.py compares it with torch.nn.GRU / nn.LSTM on CPU, forward and backward) and, through
oracle/ref_models.py, against outputs of the reference's own classes recorded in tests/golden/.

Inter-layer dropout is not modelled (compare in eval() / dropout=0, SURVEY.md §8c).

Ragged batches (``lengths``): PackedSequence semantics of the same modules (packed branch of GRU.forward /
LSTM.forward, rnn.py:1393-1394,1459-1470 / :1095-1096,1195-1206, fed by torch.nn.utils.rnn.pack_padded_sequence) on the
padded [T,B,*] block: sequence b takes lengths[b] steps (the reverse direction starts at lengths[b]-1), keeps its state
afterwards - so h_n / c_n are its state at its last valid step - and its padded output rows are 0. The reference
pads instead of packing (DAICFeatureExtarction/feature_extraction.py:45-64 produces the ragged sequences); pinned
against stock torch on packed inputs in tests/test_oracle.py.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np


def _sigmoid(x: np.ndarray) -> np.ndarray:
    return 1.0 / (1.0 + np.exp(-x))


def _gates(mode: str) -> int:
    if mode == "gru":
        return 3
    if mode == "lstm":
        return 4
    raise ValueError(mode)


def _layer_forward(mode: str, x: np.ndarray, w_ih, w_hh, b_ih, b_hh, reverse: bool, lengths=None):
    """One layer, one direction. x [T,B,I] -> y [T,B,H], final h (and c), cache for backward."""
    T, B, _ = x.shape
    live = None if lengths is None else (np.arange(T)[:, None] < np.asarray(lengths)[None, :])  # [T,B]
    H = w_hh.shape[1]
    h = np.zeros((B, H), dtype=x.dtype)
    c = np.zeros((B, H), dtype=x.dtype)
    y = np.zeros((T, B, H), dtype=x.dtype)
    cache: List[dict] = [None] * T  # type: ignore
    order = range(T - 1, -1, -1) if reverse else range(T)
    for t in order:
        gi = x[t] @ w_ih.T + b_ih
        gh = h @ w_hh.T + b_hh
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


def _layer_backward(mode: str, x, w_ih, w_hh, cache, dy, dh_last, dc_last, reverse: bool, lengths=None):
    """BPTT of one layer/direction. Returns dx, dw_ih, dw_hh, db_ih, db_hh."""
    T, B, _ = x.shape
    live = None if lengths is None else (np.arange(T)[:, None] < np.asarray(lengths)[None, :])  # [T,B]
    H = w_hh.shape[1]
    dx = np.zeros_like(x)
    dw_ih = np.zeros_like(w_ih)
    dw_hh = np.zeros_like(w_hh)
    db_ih = np.zeros(w_ih.shape[0], dtype=x.dtype)
    db_hh = np.zeros(w_ih.shape[0], dtype=x.dtype)
    dh = dh_last.copy()
    dc = dc_last.copy()
    order = range(T) if reverse else range(T - 1, -1, -1)  # reverse of the forward scan
    for t in order:
        k = cache[t]
        m = None if live is None else live[t][:, None]
        dht = dh + (dy[t] if m is None else np.where(m, dy[t], 0.0))  # a padded output row is the constant 0
        if mode == "gru":
            r, z, n, hn, h_prev = k["r"], k["z"], k["n"], k["hn"], k["h_prev"]
            dn = dht * (1.0 - z) * (1.0 - n * n)
            dz = dht * (h_prev - n) * z * (1.0 - z)
            dr = dn * hn * r * (1.0 - r)
            dgi = np.concatenate([dr, dz, dn], axis=1)
            dgh = np.concatenate([dr, dz, dn * r], axis=1)
            if m is not None:  # frozen step: no gate gradient, dh passes straight through
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
            if m is not None:  # frozen step: dh and dc pass straight through
                dgi = dgi * m
                dc = np.where(m, dct * f, dc)
                dh = np.where(m, 0.0, dht) + dgi @ w_hh
            else:
                dc = dct * f
                dh = dgi @ w_hh
            dgh = dgi
        dx[t] = dgi @ w_ih
        dw_ih += dgi.T @ x[t]
        dw_hh += dgh.T @ h_prev
        db_ih += dgi.sum(axis=0)
        db_hh += dgh.sum(axis=0)
    return dx, dw_ih, dw_hh, db_ih, db_hh


class NumpyRNN:
    """Multi-layer (bi)directional GRU/LSTM, time-major [T,B,*], with an explicit backward."""

    def __init__(self, mode: str, weights: Sequence[np.ndarray], num_layers: int, bidirectional: bool,
                 dtype=np.float64):
        self.mode = mode
        self.L = num_layers
        self.D = 2 if bidirectional else 1
        assert len(weights) == 4 * self.L * self.D
        self.w = [np.asarray(w, dtype=dtype) for w in weights]
        self.dtype = dtype
        self._saved = None

    def _p(self, l: int, d: int):
        base = 4 * (l * self.D + d)
        return self.w[base:base + 4]

    def forward(self, x: np.ndarray, lengths=None):
        """x [T,B,I] (padded); ``lengths`` [B] = valid steps per sequence (PackedSequence semantics) or None."""
        x = np.asarray(x, dtype=self.dtype)
        self._lengths = None if lengths is None else np.asarray(lengths, dtype=np.int64)
        inp = x
        h_n, c_n, saved = [], [], []
        for l in range(self.L):
            outs, caches = [], []
            for d in range(self.D):
                w_ih, w_hh, b_ih, b_hh = self._p(l, d)
                y, h, c, cache = _layer_forward(self.mode, inp, w_ih, w_hh, b_ih, b_hh, reverse=(d == 1),
                                                lengths=self._lengths)
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
        dy = np.asarray(dy, dtype=self.dtype)
        grads: Dict[Tuple[int, int], tuple] = {}
        for l in range(self.L - 1, -1, -1):
            inp, caches = self._saved[l]
            T, B, _ = inp.shape
            H = self._p(l, 0)[1].shape[1]
            dinp = np.zeros_like(inp)
            for d in range(self.D):
                w_ih, w_hh, _, _ = self._p(l, d)
                idx = l * self.D + d
                dh_last = np.zeros((B, H), self.dtype) if dh_n is None else np.asarray(dh_n[idx], self.dtype)
                dc_last = np.zeros((B, H), self.dtype) if dc_n is None else np.asarray(dc_n[idx], self.dtype)
                dyd = dy[:, :, d * H:(d + 1) * H]
                dx, dw_ih, dw_hh, db_ih, db_hh = _layer_backward(self.mode, inp, w_ih, w_hh, caches[d], dyd,
                                                                 dh_last, dc_last, reverse=(d == 1),
                                                                 lengths=self._lengths)
                dinp += dx
                grads[(l, d)] = (dw_ih, dw_hh, db_ih, db_hh)
            dy = dinp
        flat = []
        for l in range(self.L):
            for d in range(self.D):
                flat.extend(grads[(l, d)])
        return dy, flat
