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

Inter-layer dropout: ``forward(x, masks=...)`` takes the factor (0 or 1 / (1 - p)) of every element of each
layer's output but the last, [T, B, D*H] time-major - element (t*B + b)*D*H + j is what the library's dropout reads
from Philox stream l at the forward's offset (oracle/philox.py). ``backward`` applies the same factors to the gradient.

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


# ---- single steps in float64, with the magnitude each result is computed from ------------------------------------
# Each returns the next state from a given previous one and, per element of the new state, the componentwise magnitude
#   S = 1 + sum over the element's gate rows of (|b_ih| + |b_hh| + |W_ih| |x| + |W_hh| |h_prev|)
# (LSTM: + |f c_prev| + |i g|): the sum of the absolute values of every term the kernel adds up for that element. A
# floating-point evaluation of the step with unit roundoff u errs by a small multiple of u * S per element (the "1" holds
# the activations to their absolute accuracy); tests/test_gpu_numerics_f64.py states the multiple.

def _f64(*a):
    return [np.asarray(v, dtype=np.float64) for v in a]


def gru_step(x, h, w_ih, w_hh, b_ih, b_hh):
    """x [B,I], h [B,H] -> (h' [B,H], S [B,H]); torch gate order r, z, n"""
    x, h, w_ih, w_hh, b_ih, b_hh = _f64(x, h, w_ih, w_hh, b_ih, b_hh)
    H = h.shape[1]
    gi, gh = x @ w_ih.T + b_ih, h @ w_hh.T + b_hh
    r = _sigmoid(gi[:, :H] + gh[:, :H])
    z = _sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
    n = np.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
    mag = np.abs(x) @ np.abs(w_ih).T + np.abs(h) @ np.abs(w_hh).T + np.abs(b_ih) + np.abs(b_hh)  # [B, 3H]
    S = 1.0 + mag.reshape(-1, 3, H).sum(axis=1) + np.abs(h)
    return (1.0 - z) * n + z * h, S


def lstm_step(x, h, c, w_ih, w_hh, b_ih, b_hh, w_hr=None):
    """x [B,I], h [B,HO], c [B,H] -> (h' [B,HO], c' [B,H], S_h [B,HO], S_c [B,H]); gate order i, f, g, o.
    With w_hr [P,H] (proj_size = P) the new state is h' = W_hr (o tanh(c')), and S_h = 1 + |W_hr| S_m with S_m the
    magnitude of o tanh(c')."""
    x, h, c, w_ih, w_hh, b_ih, b_hh = _f64(x, h, c, w_ih, w_hh, b_ih, b_hh)
    H = c.shape[1]
    a = x @ w_ih.T + h @ w_hh.T + b_ih + b_hh
    i, f, g, o = _sigmoid(a[:, :H]), _sigmoid(a[:, H:2 * H]), np.tanh(a[:, 2 * H:3 * H]), _sigmoid(a[:, 3 * H:])
    c_new = f * c + i * g
    m = o * np.tanh(c_new)
    mag = np.abs(x) @ np.abs(w_ih).T + np.abs(h) @ np.abs(w_hh).T + np.abs(b_ih) + np.abs(b_hh)  # [B, 4H]
    S_c = 1.0 + mag.reshape(-1, 4, H).sum(axis=1) + np.abs(f * c) + np.abs(i * g)
    if w_hr is None:
        return m, c_new, S_c, S_c
    w_hr = np.asarray(w_hr, dtype=np.float64)
    return m @ w_hr.T, c_new, 1.0 + S_c @ np.abs(w_hr).T, S_c


def elman_step(x, h, w_ih, w_hh, b_ih, b_hh, nonlinearity="tanh"):
    """x [B,I], h [B,H] -> (h' [B,H], S [B,H]); h' = act(W_ih x + b_ih + W_hh h + b_hh) (torch.nn.RNN,
    rnn.py:496-505). relu is exact, so its S has no activation term: S is the magnitude of the pre-activation's terms."""
    x, h, w_ih, w_hh, b_ih, b_hh = _f64(x, h, w_ih, w_hh, b_ih, b_hh)
    a = x @ w_ih.T + b_ih + h @ w_hh.T + b_hh
    mag = np.abs(x) @ np.abs(w_ih).T + np.abs(h) @ np.abs(w_hh).T + np.abs(b_ih) + np.abs(b_hh)
    if nonlinearity == "relu":
        return np.maximum(a, 0.0), mag
    return np.tanh(a), 1.0 + mag


# ---- linearised single steps (forward-mode AD) in float64, with the magnitude each tangent is computed from ---------
# Each takes the primal (x, h[, c], W_ih, W_hh, b_ih, b_hh) and the tangents (x', h'[, c'], W_ih', W_hh', b_ih', b_hh'),
# any tangent None = 0, and returns the tangent of the new state and, per element, a magnitude S' for the bound
#   |h'_kernel - h'_64| <= KAPPA_T u S'        (tests/test_gpu_jvp_numerics_f64.py derives KAPPA_T)
# S' = R + S Q covers both error sources of a kernel that applies the linearised cell at its own saved activations:
#   R  the rounding of the tangent itself: per gate row the magnitude M of the tangent pre-activation
#      |W_ih| |x'| + |W_ih'| |x| + |W_hh| |h'| + |W_hh'| |h| + |b_ih'| + |b_hh'| (the GRU's n block: x side and h side
#      separately), each row weighted by max(1, |d state' / d row|) - the r row of the GRU is scaled by r (1 - r) |hn|,
#      the f row of the LSTM by f (1 - f) |c_prev|, either of which can exceed 1 - plus the products the linearised
#      cell adds up (GRU |(1 - z) dn|, |z h'|, |dz (h - n)|, |dr hn|, |(1 - z) (n's tangent pre-activation)|; LSTM
#      |df c|, |f c'|, |di g|, |i dg|, |do tanh c|, |o c'_t|);
#   S Q the primal's own error: the saved activations (gates, GRU hn, LSTM c_t) lie within the primal step's bound
#      KAPPA u S (gru_step / lstm_step / elman_step) of float64, and Q is the sum over those saved values of the
#      magnitude of the tangent's partial derivative with respect to each, so S Q bounds what that error moves the
#      tangent by (KAPPA <= KAPPA_T, so KAPPA_T u S' covers KAPPA u S Q).

def _dots(tangents, like):
    return [np.zeros_like(v) if t is None else np.asarray(t, dtype=np.float64) for t, v in zip(tangents, like)]


def _pre_jvp(x, h, w_ih, w_hh, xd, hd, wid, whd, bid, bhd):
    """the x-side and h-side tangent pre-activations [B, G*H] and their magnitudes"""
    ai = xd @ w_ih.T + x @ wid.T + bid
    ah = hd @ w_hh.T + h @ whd.T + bhd
    mi = np.abs(xd) @ np.abs(w_ih).T + np.abs(x) @ np.abs(wid).T + np.abs(bid)
    mh = np.abs(hd) @ np.abs(w_hh).T + np.abs(h) @ np.abs(whd).T + np.abs(bhd)
    return ai, ah, mi, mh


def gru_step_jvp(x, h, w_ih, w_hh, b_ih, b_hh, xd=None, hd=None, w_ihd=None, w_hhd=None, b_ihd=None, b_hhd=None):
    """x [B,I], h [B,H] and their tangents -> (h'_t [B,H], S' [B,H])"""
    x, h, w_ih, w_hh, b_ih, b_hh = _f64(x, h, w_ih, w_hh, b_ih, b_hh)
    xd, hd, wid, whd, bid, bhd = _dots((xd, hd, w_ihd, w_hhd, b_ihd, b_hhd), (x, h, w_ih, w_hh, b_ih, b_hh))
    H = h.shape[1]
    gi, gh = x @ w_ih.T + b_ih, h @ w_hh.T + b_hh
    r = _sigmoid(gi[:, :H] + gh[:, :H])
    z = _sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
    hn = gh[:, 2 * H:]
    n = np.tanh(gi[:, 2 * H:] + r * hn)
    _, S = gru_step(x, h, w_ih, w_hh, b_ih, b_hh)
    ai, ah, mi, mh = _pre_jvp(x, h, w_ih, w_hh, xd, hd, wid, whd, bid, bhd)
    a_r, a_z = ai[:, :H] + ah[:, :H], ai[:, H:2 * H] + ah[:, H:2 * H]
    a_n, a_hn = ai[:, 2 * H:], ah[:, 2 * H:]
    dr, dz = r * (1 - r) * a_r, z * (1 - z) * a_z
    inner = a_n + dr * hn + r * a_hn
    dn = (1 - n * n) * inner
    hdot = (1 - z) * dn + z * hd + dz * (h - n)
    m = mi + mh
    R = (m[:, :H] * np.maximum(1.0, r * (1 - r) * np.abs(hn)) + m[:, H:2 * H] + mi[:, 2 * H:] + mh[:, 2 * H:]
         + np.abs((1 - z) * dn) + np.abs(z * hd) + np.abs(dz * (h - n)) + np.abs(dr * hn) + np.abs((1 - z) * inner))
    Q = (np.abs(a_r) * np.abs(hn) + np.abs(a_hn)                          # r
         + np.abs(dn) + np.abs(hd) + np.abs(a_z) * np.abs(h - n)           # z
         + 2 * np.abs(inner) + np.abs(dz)                                   # n
         + np.abs(dr))                                                      # hn
    return hdot, R + S * Q


def lstm_step_jvp(x, h, c, w_ih, w_hh, b_ih, b_hh, xd=None, hd=None, cd=None, w_ihd=None, w_hhd=None, b_ihd=None,
                  b_hhd=None):
    """x [B,I], h [B,H], c [B,H] and their tangents -> (h'_t, c'_t, S'_h, S'_c), each [B,H]"""
    x, h, c, w_ih, w_hh, b_ih, b_hh = _f64(x, h, c, w_ih, w_hh, b_ih, b_hh)
    xd, hd, cd, wid, whd, bid, bhd = _dots((xd, hd, cd, w_ihd, w_hhd, b_ihd, b_hhd), (x, h, c, w_ih, w_hh, b_ih, b_hh))
    H = c.shape[1]
    a = x @ w_ih.T + h @ w_hh.T + b_ih + b_hh
    i, f, g, o = _sigmoid(a[:, :H]), _sigmoid(a[:, H:2 * H]), np.tanh(a[:, 2 * H:3 * H]), _sigmoid(a[:, 3 * H:])
    c_new = f * c + i * g
    tc = np.tanh(c_new)
    _, _, _, S = lstm_step(x, h, c, w_ih, w_hh, b_ih, b_hh)
    ai, ah, mi, mh = _pre_jvp(x, h, w_ih, w_hh, xd, hd, wid, whd, bid, bhd)
    ad, m = ai + ah, mi + mh
    di, df = i * (1 - i) * ad[:, :H], f * (1 - f) * ad[:, H:2 * H]
    dg, do = (1 - g * g) * ad[:, 2 * H:3 * H], o * (1 - o) * ad[:, 3 * H:]
    cdot = df * c + f * cd + di * g + i * dg
    hdot = do * tc + o * (1 - tc * tc) * cdot
    rows = (m[:, :H] + m[:, H:2 * H] * np.maximum(1.0, f * (1 - f) * np.abs(c)) + m[:, 2 * H:3 * H] + m[:, 3 * H:])
    R_c = rows + np.abs(df * c) + np.abs(f * cd) + np.abs(di * g) + np.abs(i * dg)
    R_h = R_c + np.abs(do * tc) + np.abs(o * cdot)
    Q_c = (np.abs(ad[:, :H] * g) + np.abs(dg)                               # i
           + np.abs(ad[:, H:2 * H] * c) + np.abs(cd)                        # f
           + np.abs(di) + 2 * np.abs(i * g * ad[:, 2 * H:3 * H]))           # g
    Q_h = (Q_c + np.abs(ad[:, 3 * H:] * tc) + np.abs(cdot)                  # o
           + np.abs(do) + 2 * np.abs(o * cdot))                             # c_t
    return hdot, cdot, R_h + S * Q_h, R_c + S * Q_c


def elman_step_jvp(x, h, w_ih, w_hh, b_ih, b_hh, xd=None, hd=None, w_ihd=None, w_hhd=None, b_ihd=None, b_hhd=None,
                   nonlinearity="tanh"):
    """x [B,I], h [B,H] and their tangents -> (h'_t [B,H], S' [B,H]). relu: the tangent is a' where a > 0, exact
    there, so S' carries no primal term (the branch is the precondition the caller checks)."""
    x, h, w_ih, w_hh, b_ih, b_hh = _f64(x, h, w_ih, w_hh, b_ih, b_hh)
    xd, hd, wid, whd, bid, bhd = _dots((xd, hd, w_ihd, w_hhd, b_ihd, b_hhd), (x, h, w_ih, w_hh, b_ih, b_hh))
    h_new, S = elman_step(x, h, w_ih, w_hh, b_ih, b_hh, nonlinearity)
    ai, ah, mi, mh = _pre_jvp(x, h, w_ih, w_hh, xd, hd, wid, whd, bid, bhd)
    ad, m = ai + ah, mi + mh
    if nonlinearity == "relu":
        return np.where(h_new > 0, ad, 0.0), m
    return (1 - h_new * h_new) * ad, m + S * 2 * np.abs(ad)


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

    def forward(self, x: np.ndarray, lengths=None, masks=None):
        """x [T,B,I] (padded); ``lengths`` [B] = valid steps per sequence (PackedSequence semantics) or None;
        ``masks``: L - 1 dropout factors [T,B,D*H] multiplied into the output of layers 0..L-2, or None."""
        x = np.asarray(x, dtype=self.dtype)
        self._masks = None if masks is None else [np.asarray(m, dtype=self.dtype) for m in masks]
        assert self._masks is None or len(self._masks) == self.L - 1
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
            if self._masks is not None and l < self.L - 1:
                inp = inp * self._masks[l]
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
            dy = dinp if (self._masks is None or l == 0) else dinp * self._masks[l - 1]
        flat = []
        for l in range(self.L):
            for d in range(self.D):
                flat.extend(grads[(l, d)])
        return dy, flat
