"""ORACLE — test infrastructure only (never imported by the product path).

Float64 references of the model-shell kernels, each with a componentwise error bound of the fp32 kernel:

    |out - out64| <= u * S + TINY,    u = 2^-24,  TINY = 2^-126 (results that underflow in fp32)

S is returned next to every value. It is a first-order bound that counts the kernel's rounding stages (kappa, spelled
out per function) on the float64 magnitudes, and carries the error of every earlier stage forward through the
absolute Jacobian of the later ones: a score error reaches the context through the softmax, a logit error reaches the
loss and the gradient. The worst case is taken: a chain of n roundings counts n, not sqrt(n). Library accuracies (CUDA
Programming Guide, Mathematical Functions): expf and tanhf 2 ulp, logf, expm1f and log1pf 1 ulp, rsqrtf 2 ulp; sqrtf
and division are correctly rounded (no fast-math). One ulp is up to 2u of the result (the bottom of a binade), so a
library function of k ulp counts 2k here (EXPF, TANHF, LOGF, LOG1PF, EXPM1F, RSQRTF below); a correctly rounded
operation counts 1. Second-order terms are covered by a 1 % factor.

Every function takes its inputs, and its hyperparameters, as the fp32 values the kernel receives (float32 arrays and
np.float32 scalars) and computes in float64 from there, so rounding the ABI's `float` arguments is not counted as
kernel error. Reductions follow the kernels' shapes: a warp dot over n terms is ceil(n / 32) sequential adds per lane
and a 5-level shuffle tree.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -126
SECOND_ORDER = 1.01
ULP = 2                              # u per ulp, worst case
EXPF = TANHF = RSQRTF = 2 * ULP
LOGF = LOG1PF = EXPM1F = 1 * ULP


def _f64(*xs):
    return [np.asarray(x, dtype=np.float64) for x in xs]


def warp_len(n):
    """roundings on the path of one term of a 32-lane strided sum over n terms: per-lane chain + shuffle tree"""
    return math.ceil(n / 32) + 5


def within(out, ref, S):
    """max over elements of |out - ref| / (u S + TINY): <= 1 is within the bound"""
    out, ref, S = _f64(out, ref, S)
    return float(np.max(np.abs(out - ref) / (U * S + TINY))) if out.size else 0.0


# ---- LayerNorm -----------------------------------------------------------------------------------------------------
def layernorm(x, gamma, beta, eps):
    """y = (x - mean) / sqrt(var + eps) * gamma + beta over the last axis (biased variance, nn.LayerNorm).
    Returns (y, xhat, rstd) in float64."""
    x, gamma, beta = _f64(x, gamma, beta)
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + float(eps))
    xhat = (x - mu) * rstd
    return xhat * gamma + beta, xhat, rstd


def layernorm_bwd(dy, x, gamma, eps):
    """(dx, dgamma, dbeta) of layernorm: dx = rstd (g - mean(g) - xhat mean(g xhat)), g = dy * gamma."""
    dy, x, gamma = _f64(dy, x, gamma)
    _, xhat, rstd = layernorm(x, gamma, np.zeros_like(gamma), eps)
    g = dy * gamma
    dx = rstd * (g - g.mean(-1, keepdims=True) - xhat * (g * xhat).mean(-1, keepdims=True))
    rows = dy.reshape(-1, dy.shape[-1])
    return dx, (rows * xhat.reshape(rows.shape)).sum(0), rows.sum(0)


def layernorm_bounds(x, gamma, beta, eps, dy=None, nblocks=1):
    """Bounds of layernorm_kernel / layernorm_bwd_kernel (csrc/gemm_tc.cu) on rows x [R, Cc], one warp per row, NV =
    Cc / 128 float4 per lane. Returns dict name -> (value, S): y, and with dy also dx, dgamma, dbeta (dgamma / dbeta
    without the accumulate term, which the caller adds as |old|).
      sum    (x + y) + (z + w) (2), NV sequential, the 5-level tree:        n_s = NV + 7 of |x|; / Cc exact (power of 2)
      a      x - mean (1) and the mean's error                                E_a = |a| + n_s mean|x|
      v      a * a (1), the same reduction (NV + 7), and 2 |a| E_a;  / Cc exact
      rstd   rsqrtf(var + eps): the add (1) on var + eps, half the relative error of var + eps, RSQRTF
      y      a * rstd (1), * gamma (1), + beta (1)
    backward (statistics recomputed the same way):
      xhat   a * rstd (1);  g = dy gamma (1);  sg = sum g (NV + 7);  sgx = sum g xhat (NV + 8)
      dx     rstd (g - mg - xhat mgx): the subtraction (1), xhat mgx (1), the second subtraction (1), * rstd (1)
      dgamma sum_r dy xhat: one fmaf chain of rows per lane (ceil(R / (8 nblocks)) + 1), the 8 warps of a CTA (8), the
             partials of nblocks CTAs (ceil(nblocks / 32) + 5) and the final accumulate (1);  dbeta the same without
             the product."""
    x, gamma, beta = _f64(x, gamma, beta)
    R, Cc = x.shape
    NV = Cc // 128
    ns = NV + 7
    mu = x.mean(1, keepdims=True)
    a = x - mu
    E_a = np.abs(a) + ns * np.abs(x).mean(1, keepdims=True)
    var = (a * a).mean(1, keepdims=True)
    E_var = ((ns + 1) * (a * a).sum(1, keepdims=True) + 2 * (np.abs(a) * E_a).sum(1, keepdims=True)) / Cc
    ve = var + float(eps)
    rstd = 1 / np.sqrt(ve)
    rel_r = 0.5 * (E_var + ve) / ve + RSQRTF                          # relative error of rstd, in u
    xh = a * rstd
    y = xh * gamma + beta
    E_xh = rstd * E_a + np.abs(xh) * (rel_r + 1)
    S_y = np.abs(gamma) * (E_xh + np.abs(xh)) + np.abs(y)
    k = SECOND_ORDER
    out = dict(y=(y, k * S_y))
    if dy is None:
        return out
    dy = np.asarray(dy, np.float64)
    g = dy * gamma
    E_g = np.abs(g)
    mg = g.mean(1, keepdims=True)
    E_mg = (ns * np.abs(g).sum(1, keepdims=True) + E_g.sum(1, keepdims=True)) / Cc
    mgx = (g * xh).mean(1, keepdims=True)
    E_mgx = ((ns + 1) * (np.abs(g) * np.abs(xh)).sum(1, keepdims=True)
             + (E_g * np.abs(xh) + np.abs(g) * E_xh).sum(1, keepdims=True)) / Cc
    w = g - mg - xh * mgx
    E_w = (E_g + E_mg + E_xh * np.abs(mgx) + np.abs(xh) * E_mgx + np.abs(g - mg) + np.abs(xh * mgx) + np.abs(w))
    dx = rstd * w
    S_dx = rstd * E_w + np.abs(dx) * (rel_r + 1)
    nr = math.ceil(R / (8 * nblocks)) + 8 + math.ceil(nblocks / 32) + 5 + 1
    dgamma = (dy * xh).sum(0)
    S_dg = (nr + 1) * (np.abs(dy) * np.abs(xh)).sum(0) + (np.abs(dy) * E_xh).sum(0)
    dbeta = dy.sum(0)
    S_db = nr * np.abs(dy).sum(0)
    out.update(dx=(dx, k * S_dx), dgamma=(dgamma, k * S_dg), dbeta=(dbeta, k * S_db))
    return out


# ---- attention pooling (attention_net_with_w) ----------------------------------------------------------------------
def _attention_fwd_parts(seq, h_n, w, b):
    """seq [T, B, 2H] (fwd | rev halves), h_n [NS, B, H], w [H, H], b [H]; everything the forward and the backward
    bound need, in float64, with the error magnitudes (in units of u) of each stage:

      hsum   NS - 1 sequential adds                                      E = (NS - 1) sum_k |h_n|
      qpre   warp dot over H, + bias                                      E = (warp_len(H) + 1) (|W| |hsum| + |b|) + |W| E_hsum
      h_t    fwd + rev, one rounding                                      E = |h|
      th     tanhf (2 ulp) of a rounded argument                          E = TANHF |th| + (1 - th^2) E_h
      s_t    warp dot q . th                                              E = (warp_len(H) + 1) |q| |th| + E_q |th| + |q| E_th
      a_t    expf(s - max) (EXPF, and |s - max| u from the argument), the sum over T (warp_len(T)), 1 / z (1):
             the rounding stages count a_t (EXPF + |s_t - m| + sum_u a_u (EXPF + |s_u - m|) + warp_len(T) + 1) and the score
             errors reach a_t through the softmax Jacobian, a_t (E_s,t + sum_u a_u E_s,u)
    """
    seq, h_n, w, b = _f64(seq, h_n, w, b)
    T, B, H2 = seq.shape
    H = H2 // 2
    NS = h_n.shape[0]
    hsum = h_n.sum(0)                                                # [B, H]
    E_hs = (NS - 1) * np.abs(h_n).sum(0)
    qpre = hsum @ w.T + b
    E_qp = (warp_len(H) + 1) * (np.abs(hsum) @ np.abs(w).T + np.abs(b)) + E_hs @ np.abs(w).T
    q = np.maximum(qpre, 0.0)
    h = seq[..., :H] + seq[..., H:]                                  # [T, B, H]
    E_h = np.abs(h)
    th = np.tanh(h)
    E_th = TANHF * np.abs(th) + (1 - th * th) * E_h
    s = np.einsum("bj,tbj->tb", q, th)
    E_s = ((warp_len(H) + 1) * np.einsum("bj,tbj->tb", np.abs(q), np.abs(th))
           + np.einsum("bj,tbj->tb", E_qp, np.abs(th)) + np.einsum("bj,tbj->tb", np.abs(q), E_th))
    m = s.max(0, keepdims=True)
    e = np.exp(s - m)
    a = e / e.sum(0, keepdims=True)
    r = EXPF + np.abs(s - m)
    E_a = a * (r + (a * r).sum(0, keepdims=True) + warp_len(T) + 1) + a * (E_s + (a * E_s).sum(0, keepdims=True))
    return dict(T=T, B=B, H=H, hsum=hsum, qpre=qpre, E_qp=E_qp, q=q, h=h, E_h=E_h, th=th, E_th=E_th, s=s, a=a,
                E_a=E_a)


def attention_pool(seq, h_n, w, b):
    """ctx [B, H] = sum_t a_t h_t and its bound. kappa of the last stage: h_t recomputed (1), a_t h_t (1), the
    sequential sum over T (T), the final scale by 1 / z (1):
        S = SECOND_ORDER (sum_t E_a,t |h_t| + sum_t a_t (E_h,t + (T + 2) |h_t|))"""
    P = _attention_fwd_parts(seq, h_n, w, b)
    ctx = np.einsum("tb,tbj->bj", P["a"], P["h"])
    S = (np.einsum("tb,tbj->bj", P["E_a"], np.abs(P["h"]))
         + np.einsum("tb,tbj->bj", P["a"], P["E_h"] + (P["T"] + 2) * np.abs(P["h"])))
    return ctx, SECOND_ORDER * S


def attention_pool_bwd(seq, h_n, w, b, dctx):
    """Backward of attention_pool as attention_pool_bwd_kernel computes it (recomputed forward, then)
        da_t = dctx . h_t;  ds_t = a_t (da_t - sum_u a_u da_u);  dq = sum_t ds_t th_t;
        dh_t = a_t dctx + ds_t q (1 - th_t^2)   (both halves of dseq);  dqpre = dq [qpre > 0];  dhsum = W^T dqpre.
    Returns dict of (value, S): dseq [T, B, 2H], dqpre [B, H], dhsum [B, H] (every state of dh_n), hsum [B, H].
    kappa per stage: da warp dot (warp_len(H) + 1); the a_t of the backward is e_t * (1 / z), one rounding more than the
    forward's; dot over T warp_len(T) + 1; ds two roundings; dq T + 1 sequential; dh: a dctx (1), th^2 (1), 1 - th^2
    (1), ds q (1), times (1), the add (1); dhsum two interleaved chains of H / 2 and their sum (H / 2 + 1).
    Where |qpre| is within its own bound the ReLU mask of the kernel may differ from float64's: there the whole |dq|
    enters the bound."""
    P = _attention_fwd_parts(seq, h_n, w, b)
    dctx, w = _f64(dctx, w)
    a, h, th, q, T, H = P["a"], P["h"], P["th"], P["q"], P["T"], P["H"]
    E_a = P["E_a"] + a
    E_h, E_th = P["E_h"], P["E_th"]
    E_q = P["E_qp"]
    da = np.einsum("bj,tbj->tb", dctx, h)
    E_da = (warp_len(H) + 1) * np.einsum("bj,tbj->tb", np.abs(dctx), np.abs(h)) + np.einsum("bj,tbj->tb", np.abs(dctx), E_h)
    dot = (a * da).sum(0, keepdims=True)
    E_dot = (warp_len(T) + 1) * (a * np.abs(da)).sum(0, keepdims=True) + (E_a * np.abs(da) + a * E_da).sum(0, keepdims=True)
    dd = da - dot
    ds = a * dd
    E_ds = E_a * np.abs(dd) + a * (E_da + E_dot + np.abs(dd)) + np.abs(ds)
    dq = np.einsum("tb,tbj->bj", ds, th)
    E_dq = ((T + 1) * np.einsum("tb,tbj->bj", np.abs(ds), np.abs(th))
            + np.einsum("tb,tbj->bj", E_ds, np.abs(th)) + np.einsum("tb,tbj->bj", np.abs(ds), E_th))
    om = 1 - th * th
    dh = a[..., None] * dctx[None] + ds[..., None] * q[None] * om
    E_om = th * th + om + 2 * np.abs(th) * E_th
    E_dh = (E_a[..., None] * np.abs(dctx)[None] + 2 * a[..., None] * np.abs(dctx)[None]
            + (E_ds[..., None] * np.abs(q)[None] + np.abs(ds)[..., None] * E_q[None]) * om
            + np.abs(ds)[..., None] * np.abs(q)[None] * (2 * om + E_om) + np.abs(dh))
    live = P["qpre"] > 0
    ambiguous = np.abs(P["qpre"]) <= U * E_q
    dqpre = np.where(live, dq, 0.0)
    E_dqp = np.where(ambiguous, np.abs(dq) / U + E_dq, np.where(live, E_dq, 0.0))
    dhsum = dqpre @ w
    E_dhs = (H // 2 + 1) * (np.abs(dqpre) @ np.abs(w)) + E_dqp @ np.abs(w)
    k = SECOND_ORDER
    return dict(dseq=(np.concatenate([dh, dh], -1), k * np.concatenate([E_dh, E_dh], -1)),
                dqpre=(dqpre, k * E_dqp), dhsum=(dhsum, k * E_dhs), hsum=(P["hsum"], np.zeros_like(P["hsum"])))


# ---- Dropout -> Linear -> ReLU -> Dropout --------------------------------------------------------------------------
def mlp_dropout(x, w, b, f_in, f_out, dot_len):
    """y = ReLU(W (x * f_in) + b) * f_out with the dropout factors f (scale or 0, as oracle.philox.dropout_factor gives
    them) and the bound. dot_len: roundings on the path of one product of the kernel's dot (mlp_dropout_kernel: n
    sequential fmaf; the fuse head's matvec_rows: 4 ceil(n / 128) fmaf per lane and the 5-level tree).
    kappa: x * f_in (1), the dot (dot_len), + bias (1), * f_out (1); ReLU is 1-Lipschitz and adds nothing."""
    x, w, b, f_in, f_out = _f64(x, w, b, f_in, f_out)
    xd = x * f_in
    pre = xd @ w.T + b
    y = np.maximum(pre, 0.0) * f_out
    E_pre = dot_len * (np.abs(xd) @ np.abs(w).T) + np.abs(xd) @ np.abs(w).T + np.abs(b)
    return y, SECOND_ORDER * (np.abs(f_out) * E_pre + np.abs(y)), pre


def matvec_rows_len(n):
    """roundings on a product's path in the fuse head's matvec_rows: 4-wide fmaf chunks strided by 128, the 5-level
    tree and the bias add"""
    return 4 * math.ceil(n / 128) + 6


# ---- the fuse head's output, loss and d fc_final.0.weight ---------------------------------------------------------
def _softmax2_bound(p0, p1, E0, E1):
    """2-class softmax s = softmax(p0, p1) and its bound: the larger logit's exp is 1 exactly, the other's errs by
    EXPF + |p0 - p1| u (expf and its argument), then z (1) and one division (1); logit errors enter through the
    Jacobian s0 s1 (E0 + E1)"""
    d = np.abs(p0 - p1)
    m = np.maximum(p0, p1)
    e0, e1 = np.exp(p0 - m), np.exp(p1 - m)
    z = e0 + e1
    s0, s1 = e0 / z, e1 / z
    smin = np.minimum(s0, s1)
    common = s0 * s1 * (E0 + E1) + smin * (EXPF + d)
    return (s0, s1), (common + 3 * s0, common + 3 * s1), m, z


def fuse_head_loss(tf, af, W, labels, regression=False, w_modal=None, E_tf=None, E_af=None):
    """model output, loss and dW of the fused fuse head from the features tf [B, Ht], af [B, Ha] (fp32 values, and
    their bounds E in units of u if they carry error), W [C, Ht + Ha] = fc_final.0.weight.

    classification (C = 2): logits pt = tf W[:, :Ht]^T, pa = af W[:, Ht:]^T; loss = mean_b CE(pt) + CE(pa);
      out = softmax(pt + pa); d = (softmax - onehot) / B per head; dW[c, j] = sum_b d[b, c] f[b, j].
    regression (C = 1): loss = mean_b SmoothL1(pt - y) + SmoothL1(pa - y) (beta 1); d = clamp(p - y, -1, 1) / B;
      out = ReLU(sum_j sigmoid(g_j) f_j W_j), g = w_modal f (gate), or ReLU(pt + pa) without w_modal.
    kappa: logits warp_len(F) (one fmaf chain per lane over the text and audio columns, the tree); CE row loss:
      m + logf(z) (LOGF, 2 adds) - p_y, and the loss z error (EXPF + |d|) s_min; d: the subtraction (1), 1 / B (1) and
      the product (1); the loss: row * (1 / B) (2), then a warp sum over B (warp_len(B)); dW: B sequential fmaf.
    Returns dict name -> (value, S)."""
    tf, af, W = _f64(tf, af, W)
    B, Ht = tf.shape
    Ha = af.shape[1]
    F = Ht + Ha
    E_tf = np.zeros_like(tf) if E_tf is None else np.asarray(E_tf, np.float64)
    E_af = np.zeros_like(af) if E_af is None else np.asarray(E_af, np.float64)
    f = np.concatenate([tf, af], 1)
    E_f = np.concatenate([E_tf, E_af], 1)
    Wt, Wa = W[:, :Ht], W[:, Ht:]
    nl = warp_len(F)
    pt, pa = tf @ Wt.T, af @ Wa.T                                    # [B, C]
    E_pt = nl * (np.abs(tf) @ np.abs(Wt).T) + E_tf @ np.abs(Wt).T
    E_pa = nl * (np.abs(af) @ np.abs(Wa).T) + E_af @ np.abs(Wa).T
    invB = 1.0 / B
    if not regression:
        y = np.asarray(labels).astype(np.int64)
        oh = np.stack([y == 0, y == 1], 1).astype(np.float64)
        d = np.zeros((B, 2, 2))                                      # [b, head, class]
        E_d = np.zeros_like(d)
        lrow = np.zeros(B)
        E_l = np.zeros(B)
        for k, (p, Ep) in enumerate(((pt, E_pt), (pa, E_pa))):
            (s0, s1), (Es0, Es1), m, z = _softmax2_bound(p[:, 0], p[:, 1], Ep[:, 0], Ep[:, 1])
            py = np.where(y == 0, p[:, 0], p[:, 1])
            Epy = np.where(y == 0, Ep[:, 0], Ep[:, 1])
            Em = np.where(p[:, 0] >= p[:, 1], Ep[:, 0], Ep[:, 1])
            l = m + np.log(z) - py
            lrow += l
            smin = np.minimum(s0, s1)
            E_l += (Em + Epy + LOGF * np.log(z) + smin * (EXPF + np.abs(p[:, 0] - p[:, 1])) + 2 * (np.abs(m) + np.log(z))
                     + np.abs(l))
            for c, (s, Es) in enumerate(((s0, Es0), (s1, Es1))):
                d[:, k, c] = (s - oh[:, c]) * invB
                E_d[:, k, c] = (Es + 3 * np.abs(s - oh[:, c])) * invB
        E_l += np.abs(lrow)                                          # the two heads' add
        l0, l1 = pt[:, 0] + pa[:, 0], pt[:, 1] + pa[:, 1]
        (o0, o1), (Eo0, Eo1), _, _ = _softmax2_bound(l0, l1, E_pt[:, 0] + E_pa[:, 0] + np.abs(l0),
                                                      E_pt[:, 1] + E_pa[:, 1] + np.abs(l1))
        out, E_out = np.stack([o0, o1], 1), np.stack([Eo0, Eo1], 1)
        C = 2
    else:
        y = np.asarray(labels, np.float64)
        d = np.zeros((B, 2, 1))
        E_d = np.zeros_like(d)
        lrow = np.zeros(B)
        E_l = np.zeros(B)
        for k, (p, Ep) in enumerate(((pt, E_pt), (pa, E_pa))):
            r = p[:, 0] - y
            Er = Ep[:, 0] + np.abs(r)
            ar = np.abs(r)
            l = np.where(ar < 1, 0.5 * r * r, ar - 0.5)
            lrow += l
            E_l += np.minimum(ar, 1.0) * Er + 2 * np.abs(l) + 0.5
            g = np.clip(r, -1.0, 1.0)
            d[:, k, 0] = g * invB
            E_d[:, k, 0] = (np.where(ar < 1 + U * Er, Er, 0.0) + 2 * np.abs(g)) * invB
        E_l += np.abs(lrow)
        if w_modal is not None:
            wm = np.asarray(w_modal, np.float64)
            gp = f @ wm.T
            E_gp = matvec_rows_len(F) * (np.abs(f) @ np.abs(wm).T) + E_f @ np.abs(wm).T
            sg = 1 / (1 + np.exp(-gp))
            E_sg = sg * (1 - sg) * (E_gp + EXPF + np.abs(gp)) + 2 * sg
            po = (sg * f) @ W[0]
            E_po = ((nl + 1) * (np.abs(sg * f) @ np.abs(W[0]))
                    + (E_sg * np.abs(f) + sg * E_f) @ np.abs(W[0]))
        else:
            po = pt[:, 0] + pa[:, 0]
            E_po = E_pt[:, 0] + E_pa[:, 0] + np.abs(po)
        out, E_out = np.maximum(po, 0.0)[:, None], E_po[:, None]
        C = 1
    loss = (lrow * invB).sum()
    E_loss = (E_l * invB).sum() + (warp_len(B) + 2) * (np.abs(lrow) * invB).sum()
    dW = np.zeros((C, F))
    E_dW = np.zeros((C, F))
    for c in range(C):
        dc = np.concatenate([np.repeat(d[:, 0, c:c + 1], Ht, 1), np.repeat(d[:, 1, c:c + 1], Ha, 1)], 1)
        Edc = np.concatenate([np.repeat(E_d[:, 0, c:c + 1], Ht, 1), np.repeat(E_d[:, 1, c:c + 1], Ha, 1)], 1)
        dW[c] = (dc * f).sum(0)
        E_dW[c] = B * (np.abs(dc) * np.abs(f)).sum(0) + (Edc * np.abs(f) + np.abs(dc) * E_f).sum(0)
    k = SECOND_ORDER
    return dict(out=(out, k * E_out), loss=(loss, k * E_loss), dW=(dW, k * E_dW), row_loss=(lrow, k * E_l))


# ---- Softmax -> CrossEntropyLoss (softmax_ce_kernel) ----------------------------------------------------------------
def softmax_ce(z, labels):
    """p = softmax(z); loss_b = -log softmax(p)_y; dz = p (g - sum_c p_c g_c), g = (softmax(p) - onehot) / B.
    kappa: p: expf (2) + |z - max| (argument), the warp sum (5), the division (1), and every other class's exp error
    through the sum: p_c (EXPF + 6 + |z_c - m| + sum_k p_k (EXPF + |z_k - m|)); q = softmax(p) the same with |p - max p| <= 1, and
    the p errors through its Jacobian; the row loss: max p + logf(se) (1 ulp, 2 adds) - p_y;
    g = (q - onehot) / B (2), the dot (warp sum and product, 6), dz (2).
    Returns dict name -> (value, S) for probs, row_loss, dz."""
    z = np.asarray(z, np.float64)
    y = np.asarray(labels).astype(np.int64)
    B, C = z.shape
    m = z.max(1, keepdims=True)
    e = np.exp(z - m)
    p = e / e.sum(1, keepdims=True)
    r = EXPF + np.abs(z - m)
    E_p = p * (r + (p * r).sum(1, keepdims=True) + 6)
    m2 = p.max(1, keepdims=True)
    e2 = np.exp(p - m2)
    se = e2.sum(1, keepdims=True)
    q = e2 / se
    r2 = EXPF + np.abs(p - m2)
    E_q = q * (r2 + (q * r2).sum(1, keepdims=True) + 6) + q * (E_p + (q * E_p).sum(1, keepdims=True))
    oh = np.zeros_like(z)
    oh[np.arange(B), y] = 1.0
    py = p[np.arange(B), y]
    loss = m2[:, 0] + np.log(se[:, 0]) - py
    E_m2 = E_p[np.arange(B), p.argmax(1)]
    E_loss = (E_m2 + E_p[np.arange(B), y] + (q * (E_p + r2)).sum(1) + 6 + LOGF * np.log(se[:, 0])
              + 2 * (m2[:, 0] + np.log(se[:, 0])) + np.abs(loss))
    g = (q - oh) / B
    E_g = (E_q + 2 * np.abs(q - oh)) / B
    dot = (p * g).sum(1, keepdims=True)
    E_dot = 6 * (p * np.abs(g)).sum(1, keepdims=True) + (E_p * np.abs(g) + p * E_g).sum(1, keepdims=True)
    gd = g - dot
    dz = p * gd
    E_dz = E_p * np.abs(gd) + p * (E_g + E_dot + np.abs(gd)) + np.abs(dz)
    k = SECOND_ORDER
    return dict(probs=(p, k * E_p), row_loss=(loss, k * E_loss), dz=(dz, k * E_dz))


def mean_rows(row_loss, S_row):
    """loss = mean of the row losses as mean_rows_kernel sums them: 256 threads, each ceil(B / 256) rows in sequence
    (the first add from 0 is exact, the rest round), a 5-level warp tree, the 8 warp sums through a second 5-level
    tree, then / B (1):  S = mean S_row + (ceil(B / 256) + 11) mean |row_loss|."""
    rl, S_row = _f64(row_loss, S_row)
    B = rl.size
    return rl.mean(), SECOND_ORDER * (S_row.mean() + (math.ceil(B / 256) + 11) * np.abs(rl).mean())


# ---- Adam / AdamW (adam_update in csrc/misc_kernels.cuh) ----------------------------------------------------------
def adam(p, g, m, v, t, lr, beta1, beta2, eps, weight_decay=0.0, grad_scale=1.0):
    """One torch.optim.AdamW step (Adam at weight_decay 0) at step t (1-based), all scalars the fp32 values the kernel
    receives. Returns dict name -> (value, S) for p, m, v.

    The kernel's stages, and kappa:
      g' = g * grad_scale              exact for the power-of-two scales used (1 / world)
      m' = b1 m + (1 - b1) g'          1 - b1 exact; (1 - b1) g' (1), the fmaf (1):       S_m = 2 (|b1 m| + |(1-b1) g'|)
      v' = b2 v + (1 - b2) g'^2        two products (2), the fmaf (1):                    S_v = 3 (|b2 v| + (1-b2) g'^2)
      bc = -expm1f(t log1pf(-(1-b)))   log1pf (LOG1PF), the product (1), expm1f (EXPM1F) on an argument whose relative
                                       error it passes on times |x e^x / (e^x - 1)| <= 1:  BC = 5 u of bc
      step_size = lr / bc1             BC + 1 = 6;   rsqrtf(bc2): RSQRTF + BC / 2 = 6.5
      den = sqrtf(v') r + eps          the v' error halved, sqrtf (1), the product (1), r (3.5), the add (1)
      upd = step_size m' / den         the product (1) and the division (1)
      p' = p decay - upd               the final rounding (1) of |p'|; with weight decay also decay = 1 - lr wd
                                       (its rounding near 1 is u / 2, of |p|; lr wd (1) of |lr wd p|) and, if
                                       not fused, the product p decay (1); at wd = 0, decay = 1 and p decay = p exactly
    so |upd| carries 6 + 2 + (den - eps) / den (S_v / (2 v') + 8.5) + 1 (the eps add) relative units, and the m' error
    step_size S_m / den.
    At wd = 0 and p = 0 the output is -upd itself, so the bound is not hidden by the rounding of p."""
    p, g, m, v = _f64(p, g, m, v)
    b1, b2, lr, eps, wd, gs = (float(np.float32(x)) for x in (beta1, beta2, lr, eps, weight_decay, grad_scale))
    t = float(t)
    gg = g * gs
    mn = b1 * m + (1 - b1) * gg
    vn = b2 * v + (1 - b2) * gg * gg
    S_m = 2 * (np.abs(b1 * m) + np.abs((1 - b1) * gg))
    S_v = 3 * (np.abs(b2 * v) + (1 - b2) * gg * gg)
    bc1 = -math.expm1(t * math.log1p(-(1 - b1)))
    bc2 = -math.expm1(t * math.log1p(-(1 - b2)))
    step = lr / bc1
    root = np.sqrt(vn) / math.sqrt(bc2)
    den = root + eps
    upd = step * mn / den
    decay = 1 - lr * wd
    pn = p * decay - upd
    with np.errstate(divide="ignore", invalid="ignore"):
        rel_v = np.where(vn > 0, S_v / (2 * vn), 0.0)
    BC = LOG1PF + 1 + EXPM1F
    S_upd = np.abs(upd) * ((BC + 1) + 2 + 1 + root / den * (rel_v + RSQRTF + BC / 2 + 2)) + step * S_m / den
    S_p = S_upd + np.abs(pn)
    if wd:
        S_p = S_p + 0.5 * np.abs(p) + np.abs(lr * wd * p) + np.abs(p * decay)
    k = SECOND_ORDER
    return dict(p=(pn, k * S_p), m=(mn, k * S_m), v=(vn, k * S_v))


def adam_bias_correction_f32_pow(beta, t):
    """1 - beta^t as the fp32 expression 1.f - powf(beta, t) with a correctly rounded powf: the cancellation the
    kernels avoid (the value the previous code computed at best)"""
    pw = np.float32(float(np.float32(beta)) ** float(t))
    return float(np.float32(np.float32(1.0) - pw))
