"""The model-shell kernels against float64, element by element, under the rounding bounds of oracle/shell_numpy.py,
and every dropout mask against oracle/philox.py bit for bit.

    |out - out64| <= u S + TINY   for every output element,   u = 2^-24

Covered: Adam / AdamW (adam_kernel and the fuse head's in-kernel update, which must agree bit for bit), Softmax ->
CrossEntropy (softmax_ce_kernel), attention pooling forward and backward, Dropout-Linear-ReLU-Dropout
(mlp_dropout_kernel), the fused fuse head stage by stage (its own fp32 output of each stage feeds the oracle of the
next), and the inter-layer dropout of the GRU / LSTM (dropout_kernel). Every case is run twice and must repeat bit
for bit. The largest err / bound ratio of each case is written to $SHELL_F64_RESULTS (a JSON file) when that is set.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import philox
from oracle import shell_numpy as sh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NUM_SMS = 132
RESULTS = {}


@pytest.fixture(scope="module", autouse=True)
def _write_results():
    yield
    path = os.environ.get("SHELL_F64_RESULTS")
    if path and RESULTS:
        import subprocess

        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip().splitlines()
        name, power = (q[0].split(", ") + ["?"])[:2] if q else ("unknown", "unknown")
        with open(path, "w") as f:
            json.dump({"device": {"gpu": name, "power_limit": power}, "max_err_over_bound": RESULTS}, f, indent=1,
                      sort_keys=True)
            f.write("\n")


def _lib():
    from b200rnn import _lib as L

    return L, L.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check(case, name, out, ref, S):
    out = out.detach().double().cpu().numpy() if torch.is_tensor(out) else np.asarray(out, np.float64)
    r = sh.within(out, ref, S)
    key = f"{case}/{name}"
    RESULTS[key] = max(RESULTS.get(key, 0.0), r)
    assert np.isfinite(out).all() or not np.isfinite(ref).all(), key
    assert r <= 1.0, f"{key}: max |err| / bound = {r:.3g}"


def _d(x):
    return torch.as_tensor(np.ascontiguousarray(x), device=DEV)


# ---- Adam / AdamW -----------------------------------------------------------------------------------------------------
def _adamw(p, g, m, v, step, lr, b1, b2, eps, wd, gs, advance=1):
    L, lib = _lib()
    L.check(lib.b200rnn_adamw(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), step.data_ptr(), p.numel(), lr,
                              b1, b2, eps, wd, gs, advance, _stream()), "adamw")


@pytest.mark.parametrize("n", [1, 255, 257, NUM_SMS * 8 * 256 + 37])
@pytest.mark.parametrize("t", [1, 2, 5, 1000])
@pytest.mark.parametrize("wd,gs", [(0.0, 1.0), (1e-2, 0.125)])
def test_adamw_update_within_bound(n, t, wd, gs):
    """p = 0, so the output is the update itself; g = 0 and v << eps^2 in part of the range; t counted on the device"""
    rng = np.random.default_rng(n + t)
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    g = rng.standard_normal(n).astype(np.float32) * np.float32(1e-3)
    m = rng.standard_normal(n).astype(np.float32) * np.float32(1e-4)
    v = (rng.standard_normal(n).astype(np.float32) * np.float32(1e-3)) ** 2
    g[::7] = 0.0
    v[::5] = np.float32(1e-20)                                   # sqrt(v) << eps
    p = np.zeros(n, np.float32)
    if wd:
        p[1::2] = rng.standard_normal(n // 2).astype(np.float32)   # the decay term on half the elements
    outs = []
    for _ in range(2):
        P, G, M, V = _d(p), _d(g), _d(m), _d(v)
        step = torch.tensor(float(t - 1), device=DEV)
        _adamw(P, G, M, V, step, lr, b1, b2, eps, wd, gs)
        torch.cuda.synchronize()
        assert step.item() == float(t)
        outs.append((P.cpu(), M.cpu(), V.cpu()))
    assert all(torch.equal(a, b) for a, b in zip(*outs)), "bitwise repeatable"
    ref = sh.adam(p, g, m, v, t, np.float32(lr), np.float32(b1), np.float32(b2), np.float32(eps), np.float32(wd), gs)
    case = f"adamw/n{n}-t{t}-wd{wd}-gs{gs}"
    for name, got in zip(("p", "m", "v"), outs[0]):
        _check(case, name, got, *ref[name])


def test_adamw_two_groups_share_one_step_counter():
    """advance_step = 0 for the first group, 1 for the last: both groups see the same t, the counter moves once"""
    rng = np.random.default_rng(3)
    lr, b1, b2, eps = 6e-6, 0.9, 0.999, 1e-8
    groups = [(rng.standard_normal(300).astype(np.float32), 1e-2), (rng.standard_normal(40).astype(np.float32), 0.0)]
    state = [(_d(np.zeros_like(g)), _d(np.zeros_like(g)), _d(np.zeros_like(g))) for g, _ in groups]
    step = torch.zeros((), device=DEV)
    host = [(np.zeros_like(g), np.zeros_like(g), np.zeros_like(g)) for g, _ in groups]
    for t in range(1, 4):
        for k, ((g, wd), (P, M, V)) in enumerate(zip(groups, state)):
            _adamw(P, _d(g), M, V, step, lr, b1, b2, eps, wd, 1.0, advance=int(k == len(groups) - 1))
        torch.cuda.synchronize()
        assert step.item() == float(t)
        for k, ((g, wd), (P, M, V)) in enumerate(zip(groups, state)):
            r = sh.adam(*host[k][:1], g, *host[k][1:], t, np.float32(lr), np.float32(b1), np.float32(b2),
                        np.float32(eps), np.float32(wd), 1.0)
            for name, got in zip(("p", "m", "v"), (P, M, V)):
                _check(f"adamw_groups/g{k}-t{t}", name, got, *r[name])
            host[k] = (P.cpu().numpy(), M.cpu().numpy(), V.cpu().numpy())


# ---- Softmax -> CrossEntropy -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 2, 31, 32])
@pytest.mark.parametrize("B", [1, 7, 8, 9, 4096])
@pytest.mark.parametrize("regime", ["normal", "saturated"])
def test_softmax_ce_within_bound(C, B, regime):
    L, lib = _lib()
    rng = np.random.default_rng(C * 10000 + B)
    z = rng.standard_normal((B, C)).astype(np.float32)
    if regime == "saturated":
        z = np.where(rng.random((B, C)) < 0.5, np.float32(-80), np.float32(80)) + z
    y = rng.integers(0, C, B).astype(np.int64)
    outs = []
    for _ in range(2):
        Z, Y = _d(z), _d(y)
        probs, dz, rl = (torch.empty(B, C, device=DEV), torch.empty(B, C, device=DEV), torch.empty(B, device=DEV))
        loss = torch.empty((), device=DEV)
        L.check(lib.b200rnn_softmax_ce(Z.data_ptr(), Y.data_ptr(), B, C, probs.data_ptr(), dz.data_ptr(), rl.data_ptr(),
                                       loss.data_ptr(), _stream()), "softmax_ce")
        torch.cuda.synchronize()
        outs.append((probs.cpu(), dz.cpu(), rl.cpu(), loss.cpu()))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    ref = sh.softmax_ce(z, y)
    case = f"softmax_ce/C{C}-B{B}-{regime}"
    _check(case, "probs", outs[0][0], *ref["probs"])
    _check(case, "dz", outs[0][1], *ref["dz"])
    _check(case, "row_loss", outs[0][2], *ref["row_loss"])
    _check(case, "loss", outs[0][3], *sh.mean_rows(*ref["row_loss"]))


# ---- attention pooling --------------------------------------------------------------------------------------------------
def _attention_inputs(T, B, H, NS, regime, seed):
    rng = np.random.default_rng(seed)
    big = np.zeros((T, B + 1, 2 * H + 8), np.float32)              # seq is a strided view: batch stride 2H + 8, row gap
    big[:, :B, :2 * H] = rng.standard_normal((T, B, 2 * H)).astype(np.float32) * np.float32(0.5)
    h_n = rng.standard_normal((NS, B, H)).astype(np.float32) * np.float32(0.5)
    w = (rng.standard_normal((H, H)) / math.sqrt(H * NS)).astype(np.float32)
    b = (rng.standard_normal(H) * 0.1).astype(np.float32)
    if regime == "sharp":                                          # scores of +-50: a (nearly) one-hot softmax
        w = w * np.float32(200 / math.sqrt(H))
    return big, h_n, w, b


ATT_CASES = [(1, 3, 4, 1), (31, 2, 20, 2), (32, 2, 64, 4), (33, 2, 128, 2), (5, 4, 256, 4), (17, 2, 512, 1),
             (47 * 256 - 2 * 64, 2, 64, 2), (47 * 256 - 2 * 64 + 1, 2, 64, 2), (95, 2, 512, 2), (192, 2, 256, 1)]


@pytest.mark.parametrize("T,B,H,NS", ATT_CASES)
@pytest.mark.parametrize("regime", ["normal", "sharp"])
def test_attention_pool_fwd_bwd_within_bound(T, B, H, NS, regime):
    L, lib = _lib()
    big, h_n, w, b = _attention_inputs(T, B, H, NS, regime, T * 7 + H)
    seq = big[:, :B, :2 * H]
    fwd_ok = (2 * H + T) * 4 <= 47 * 1024                        # 1 KB of the 48 KB stays for static shared memory
    bwd_ok = (4 * H + 2 * T + T * H) * 4 <= 200 * 1024
    BIG, HN, W, Bb = _d(big), _d(h_n), _d(w), _d(b)
    s_t, s_b = BIG.stride(0), BIG.stride(1)
    dctx = np.random.default_rng(1).standard_normal((B, H)).astype(np.float32)
    DC = _d(dctx)
    outs = []
    for _ in range(2):
        ctx = torch.empty(B, H, device=DEV)
        rc = lib.b200rnn_attention_pool(BIG.data_ptr(), s_t, s_b, HN.data_ptr(), NS, B, T, H, W.data_ptr(),
                                        Bb.data_ptr(), ctx.data_ptr(), _stream())
        if not fwd_ok:
            assert rc != 0
            return
        L.check(rc, "attention_pool")
        res = [ctx]
        if bwd_ok:
            dseq = torch.full((T, B, 2 * H), float("nan"), device=DEV)
            dhn, dqp, hs = torch.empty(NS, B, H, device=DEV), torch.empty(B, H, device=DEV), torch.empty(B, H, device=DEV)
            L.check(lib.b200rnn_attention_pool_bwd(BIG.data_ptr(), s_t, s_b, HN.data_ptr(), NS, B, T, H, W.data_ptr(),
                                                   Bb.data_ptr(), DC.data_ptr(), dseq.data_ptr(), dseq.stride(0),
                                                   dseq.stride(1), dhn.data_ptr(), dqp.data_ptr(), hs.data_ptr(),
                                                   _stream()), "attention_pool_bwd")
            res += [dseq, dhn, dqp, hs]
        torch.cuda.synchronize()
        outs.append([r.cpu() for r in res])
    assert all(torch.equal(a, c) for a, c in zip(*outs))
    case = f"attention/T{T}-B{B}-H{H}-NS{NS}-{regime}"
    ctx_ref, S = sh.attention_pool(seq, h_n, w, b)
    _check(case, "ctx", outs[0][0], ctx_ref, S)
    if bwd_ok:
        r = sh.attention_pool_bwd(seq, h_n, w, b, dctx)
        _check(case, "dseq", outs[0][1], *r["dseq"])
        for k in range(NS):
            _check(case, "dh_n", outs[0][2][k], *r["dhsum"])
        _check(case, "dqpre", outs[0][3], *r["dqpre"])
        _check(case, "hsum", outs[0][4], r["hsum"][0], (NS - 1) * np.abs(h_n).sum(0))


def test_attention_pool_rejects_the_first_shape_past_48kb_and_the_module_path_falls_back():
    """H = 64: T = 12160 (2H + T floats = 48 KB) used to be accepted and then fail at launch, because the kernel's
    static shared memory comes on top. The dynamic budget is 47 KB now: T = 11904 runs the kernel, T = 11905 and
    12160 return UNSUPPORTED, and attention_pool_tm takes the PyTorch expression for them"""
    from b200rnn import fused_head

    L, lib = _lib()
    H, B, NS = 64, 2, 2
    for T, ok in ((11904, True), (11905, False), (12160, False)):
        big, h_n, w, b = _attention_inputs(T, B, H, NS, "normal", 3)
        X, HN, Wd, Bd = _d(big), _d(h_n), _d(w), _d(b)
        ctx = torch.empty(B, H, device=DEV)
        rc = lib.b200rnn_attention_pool(X.data_ptr(), X.stride(0), X.stride(1), HN.data_ptr(), NS, B, T, H, Wd.data_ptr(),
                                        Bd.data_ptr(), ctx.data_ptr(), _stream())
        torch.cuda.synchronize()
        assert (rc == 0) == ok, (T, rc, lib.b200rnn_last_error())
        layer = torch.nn.Sequential(torch.nn.Linear(H, H), torch.nn.ReLU()).to(DEV)
        with torch.no_grad():
            layer[0].weight.copy_(Wd)
            layer[0].bias.copy_(Bd)
            got = fused_head.attention_pool_tm(layer, _d(np.ascontiguousarray(big[:, :B, :2 * H])), HN)
        ref, _ = sh.attention_pool(big[:, :B, :2 * H], h_n, w, b)
        assert np.linalg.norm(got.double().cpu().numpy() - ref) <= 1e-5 * np.linalg.norm(ref)


@pytest.mark.parametrize("T,fits", [(95, True), (96, False)])
def test_attention_pool_tm_kernel_and_fallback_at_the_limit(T, fits):
    """H = 512: T = 95 is the largest T whose backward fits one CTA, so attention_pool_tm runs the kernels (forward and
    backward launch); T = 96 takes the PyTorch expression and launches nothing of the library. Both against float64."""
    from b200rnn import fused_head

    L, lib = _lib()
    H, B, NS = 512, 2, 2
    big, h_n, w, b = _attention_inputs(T, B, H, NS, "normal", 5)
    seq = big[:, :B, :2 * H]
    layer = torch.nn.Sequential(torch.nn.Linear(H, H), torch.nn.ReLU()).to(DEV)
    with torch.no_grad():
        layer[0].weight.copy_(_d(w))
        layer[0].bias.copy_(_d(b))
    S_ = _d(np.ascontiguousarray(seq)).requires_grad_(True)
    HN = _d(h_n).requires_grad_(True)
    dctx = np.random.default_rng(2).standard_normal((B, H)).astype(np.float32)
    n0 = lib.b200rnn_launch_count()
    ctx = fused_head.attention_pool_tm(layer, S_, HN)
    (ctx * _d(dctx)).sum().backward()
    torch.cuda.synchronize()
    launched = lib.b200rnn_launch_count() - n0
    assert (launched >= 2) if fits else (launched == 0), launched
    ref, S = sh.attention_pool(seq, h_n, w, b)
    bw = sh.attention_pool_bwd(seq, h_n, w, b, dctx)
    if fits:
        _check(f"attention_tm/T{T}-H{H}", "ctx", ctx, ref, S)
        _check(f"attention_tm/T{T}-H{H}", "dseq", S_.grad, *bw["dseq"])
    else:  # torch's fp32 expression: normwise
        assert np.linalg.norm(ctx.detach().double().cpu().numpy() - ref) <= 1e-5 * np.linalg.norm(ref)
        g = S_.grad.double().cpu().numpy()
        assert np.linalg.norm(g - bw["dseq"][0]) <= 1e-4 * np.linalg.norm(bw["dseq"][0])


# ---- Dropout-Linear-ReLU-Dropout, and its two Philox streams -------------------------------------------------------------
@pytest.mark.parametrize("B,n,p", [(1, 4, 0.3), (33, 20, 0.5), (64, 256, 0.3), (7, 130, 1.0)])
def test_mlp_dropout_masks_exact_and_values_within_bound(B, n, p):
    L, lib = _lib()
    rng = np.random.default_rng(B * n)
    x = rng.standard_normal((B, n)).astype(np.float32)
    w = (rng.standard_normal((n, n)) / math.sqrt(n)).astype(np.float32)
    b = (rng.standard_normal(n) * 0.1).astype(np.float32)
    seed, off, stream = 0x1234ABCD5678, 1000003, 4
    hdr = torch.tensor([seed, off], dtype=torch.int64, device=DEV)
    X, Wd, Bd = _d(x), _d(w), _d(b)                             # held: a freed temporary's memory would be reused
    outs = []
    for _ in range(2):
        out = torch.empty(B, n, device=DEV)
        L.check(lib.b200rnn_mlp_dropout(X.data_ptr(), B, n, Wd.data_ptr(), Bd.data_ptr(), out.data_ptr(), 1,
                                        p, hdr.data_ptr(), stream, _stream()), "mlp_dropout")
        torch.cuda.synchronize()
        outs.append(out.cpu())
    assert torch.equal(*outs)
    f_in = philox.dropout_factor(seed, off, stream, B * n, p).reshape(B, n)
    f_out = philox.dropout_factor(seed, off, stream + 1, B * n, p).reshape(B, n)
    y, S, pre = sh.mlp_dropout(x, w, b, f_in, f_out, n + 1)
    got = outs[0].numpy()
    assert ((got != 0) <= (f_out != 0)).all(), "an element the output mask drops is nonzero"
    _check(f"mlp_dropout/B{B}-n{n}-p{p}", "out", got, y, S)


# ---- the fused fuse head, stage by stage -----------------------------------------------------------------------------------
class _Head:
    """host inputs of one b200rnn_fuse_head case and the argument block"""

    def __init__(self, B, Ht, Ha, T, regression, modal, seed, logit_scale=1.0):
        rng = np.random.default_rng(seed)
        self.B, self.Ht, self.Ha, self.T, self.reg = B, Ht, Ha, T, regression
        F = Ht + Ha
        C = 1 if regression else 2
        f32 = np.float32
        self.seq = (rng.standard_normal((T, B, 2 * Ht)) * 0.5).astype(f32) if T else None
        self.h_n = (rng.standard_normal((2, B, Ht)) * 0.5).astype(f32)
        self.w_att = (rng.standard_normal((Ht, Ht)) / math.sqrt(2 * Ht)).astype(f32)
        self.b_att = (rng.standard_normal(Ht) * 0.1).astype(f32)
        self.ctx = rng.standard_normal((B, Ht)).astype(f32)
        self.pooled = rng.standard_normal((B, Ha)).astype(f32)
        self.w_t = (rng.standard_normal((Ht, Ht)) / math.sqrt(Ht)).astype(f32)
        self.b_t = (rng.standard_normal(Ht) * 0.1).astype(f32)
        self.w_a = (rng.standard_normal((Ha, Ha)) / math.sqrt(Ha)).astype(f32)
        self.b_a = (rng.standard_normal(Ha) * 0.1).astype(f32)
        self.W = (rng.standard_normal((C, F)) * logit_scale / math.sqrt(F)).astype(f32)
        self.w_modal = (rng.standard_normal((F, F)) / math.sqrt(F)).astype(f32) if modal else None
        self.labels = ((rng.random(B) * 3).astype(f32) if regression else rng.integers(0, 2, B).astype(np.int64))
        self.dev = {k: _d(v) for k, v in vars(self).items() if isinstance(v, np.ndarray)}

    def run(self, training, p, seed, offset, loss=True, adam=True, t0=0, tf_in=None):
        L, lib = _lib()
        B, Ht, Ha, F = self.B, self.Ht, self.Ha, self.Ht + self.Ha
        C = 1 if self.reg else 2
        D = self.dev
        o = dict(tf=torch.empty(B, Ht, device=DEV), af=torch.empty(B, Ha, device=DEV),
                 ctx=torch.empty(B, Ht, device=DEV), rng=torch.tensor([seed, offset], dtype=torch.int64, device=DEV))
        a = L.FuseHeadArgs(B=B, T=self.T, Ht=Ht, Ha=Ha, n_states=2, training=int(training), p=p,
                           regression=int(self.reg), pooled=D["pooled"].data_ptr(), w_a=D["w_a"].data_ptr(),
                           b_a=D["b_a"].data_ptr(), w_t=D["w_t"].data_ptr(), b_t=D["b_t"].data_ptr(),
                           text_feature=o["tf"].data_ptr(), audio_feature=o["af"].data_ptr(),
                           rng_state=o["rng"].data_ptr(), rng_consume=(B * max(Ht, Ha) + 3) // 4)
        if tf_in is not None:
            a.tf_in, a.text_feature = tf_in.data_ptr(), None
        elif self.T:
            a.seq, a.seq_st, a.seq_sb = D["seq"].data_ptr(), B * 2 * Ht, 2 * Ht
            a.h_n, a.w_att, a.b_att, a.ctx_out = D["h_n"].data_ptr(), D["w_att"].data_ptr(), D["b_att"].data_ptr(), o["ctx"].data_ptr()
        else:
            a.ctx_in = D["ctx"].data_ptr()
        if loss:
            o.update(W=D["W"].clone(), out=torch.empty(B, C, device=DEV), loss=torch.empty((), device=DEV),
                     dw=torch.zeros(C * F + 1, device=DEV), ticket=torch.zeros(1, dtype=torch.int32, device=DEV),
                     dw_part=torch.empty(int(lib.b200rnn_fuse_head_scratch_floats(B, Ht, Ha, int(self.reg))), device=DEV),
                     m=_d(np.full(C * F, 1e-3, np.float32)), v=_d(np.full(C * F, 1e-6, np.float32)),
                     step=torch.tensor(float(t0), device=DEV))
            a.W, a.out, a.loss, a.dw = o["W"].data_ptr(), o["out"].data_ptr(), o["loss"].data_ptr(), o["dw"].data_ptr()
            a.labels, a.dw_part, a.ticket = D["labels"].data_ptr(), o["dw_part"].data_ptr(), o["ticket"].data_ptr()
            a.w_modal = D["w_modal"].data_ptr() if self.w_modal is not None else None
            a.do_adam, a.adam_m, a.adam_v, a.adam_step = int(adam), o["m"].data_ptr(), o["v"].data_ptr(), o["step"].data_ptr()
            a.lr, a.beta1, a.beta2, a.eps, a.grad_scale, a.world = 1e-3, 0.9, 0.999, 1e-8, 1.0, 1
        rc = lib.b200rnn_fuse_head(__import__("ctypes").byref(a), _stream())
        torch.cuda.synchronize()
        return rc, {k: v.cpu() if torch.is_tensor(v) else v for k, v in o.items()}


HEAD_CASES = [  # B, Ht, Ha, T, regression, modal
    (1, 4, 12, 0, False, False), (15, 12, 4, 0, True, True), (17, 64, 128, 0, False, False),
    (16, 128, 256, 0, True, False), (128, 128, 256, 0, False, False), (1000, 256, 128, 0, False, False),
    (8, 512, 512, 0, True, True), (5, 128, 256, 7, False, False), (3, 20, 12, 33, True, True),
]


@pytest.mark.parametrize("B,Ht,Ha,T,reg,modal", HEAD_CASES)
@pytest.mark.parametrize("p", [0.0, 0.3, 0.5, 1.0])
def test_fuse_head_stages_and_masks_within_bound(B, Ht, Ha, T, reg, modal, p):
    """teacher-forced: the context (given, or the kernel's own ctx_out) -> the features with the kernel's masks of
    streams 0..3 from oracle.philox; the kernel's features -> out, loss, dW; the kernel's dW -> W, m, v"""
    h = _Head(B, Ht, Ha, T, reg, modal, seed=B * 131 + Ht + T)
    seed, off = 0x5DEECE66D + B, 12345 + Ht
    train = p > 0
    rc, r = h.run(train, p, seed, off, t0=4)
    L, _ = _lib()
    L.check(rc, "fuse_head")
    rc2, r2 = h.run(train, p, seed, off, t0=4)
    for k in ("tf", "af", "out", "loss", "dw", "W", "m", "v"):
        assert torch.equal(r[k], r2[k]), k
    assert r["rng"][1].item() == (off + (B * max(Ht, Ha) + 3) // 4 if train else off), "offset advances by rng_consume"
    case = f"fuse_head/B{B}-Ht{Ht}-Ha{Ha}-T{T}-{'reg' if reg else 'cls'}{'-modal' if modal else ''}-p{p}"
    fac = (lambda s, n: philox.dropout_factor(seed, off, s, B * n, p).reshape(B, n)) if train else \
          (lambda s, n: np.ones((B, n), np.float32))
    if T:
        ctx_ref, S = sh.attention_pool(h.seq, h.h_n, h.w_att, h.b_att)
        _check(case, "ctx_out", r["ctx"], ctx_ref, S)
        ctx_in = r["ctx"].numpy()
    else:
        ctx_in = h.ctx
    tf_ref, S_tf, _ = sh.mlp_dropout(ctx_in, h.w_t, h.b_t, fac(0, Ht), fac(1, Ht), sh.matvec_rows_len(Ht))
    af_ref, S_af, _ = sh.mlp_dropout(h.pooled, h.w_a, h.b_a, fac(2, Ha), fac(3, Ha), sh.matvec_rows_len(Ha))
    if train:
        assert ((r["tf"].numpy() != 0) <= (fac(1, Ht) != 0)).all() and ((r["af"].numpy() != 0) <= (fac(3, Ha) != 0)).all()
    _check(case, "text_feature", r["tf"], tf_ref, S_tf)
    _check(case, "audio_feature", r["af"], af_ref, S_af)
    tf, af = r["tf"].numpy(), r["af"].numpy()
    ref = sh.fuse_head_loss(tf, af, h.W, h.labels, regression=reg, w_modal=h.w_modal)
    C = 1 if reg else 2
    F = Ht + Ha
    _check(case, "out", r["out"], *ref["out"])
    _check(case, "loss", r["loss"], *ref["loss"])
    _check(case, "dw", r["dw"][:C * F].view(C, F), *ref["dW"])
    dw = r["dw"][:C * F].numpy()
    a = sh.adam(h.W.reshape(-1), dw, np.full(C * F, 1e-3, np.float32), np.full(C * F, 1e-6, np.float32), 5,
                np.float32(1e-3), np.float32(0.9), np.float32(0.999), np.float32(1e-8))
    _check(case, "W", r["W"].view(-1), *a["p"])
    _check(case, "m", r["m"], *a["m"])
    _check(case, "v", r["v"], *a["v"])


@pytest.mark.parametrize("regime", ["logits60", "smoothl1_knee", "smoothl1_far"])
def test_fuse_head_loss_saturated_regimes(regime):
    """logits of +-60 (CE in its linear tail), SmoothL1 residuals at 1 +- 2^-20 (the knee) and >> 1"""
    reg = regime != "logits60"
    h = _Head(64, 128, 256, 0, reg, False, seed=7, logit_scale=70.0 if not reg else 1.0)
    _, r0 = h.run(False, 0.0, 1, 0, loss=False)
    tf, af = r0["tf"].numpy().astype(np.float64), r0["af"].numpy().astype(np.float64)
    if reg:
        pt = tf @ h.W[0, :128].astype(np.float64)
        sgn = np.where(np.arange(64) % 2 == 0, 1.0, -1.0)
        d = (1 + sgn * 2.0 ** -20) if regime == "smoothl1_knee" else 40.0 * sgn
        h.labels = (pt - d).astype(np.float32)
        h.dev["labels"] = _d(h.labels)
    _, r = h.run(False, 0.0, 1, 0)
    ref = sh.fuse_head_loss(r["tf"].numpy(), r["af"].numpy(), h.W, h.labels, regression=reg)
    C = 1 if reg else 2
    case = f"fuse_head_regime/{regime}"
    if not reg:
        assert np.abs(tf @ h.W.T[:128].astype(np.float64)).max() > 30
    _check(case, "out", r["out"], *ref["out"])
    _check(case, "loss", r["loss"], *ref["loss"])
    _check(case, "dw", r["dw"][:C * 384].view(C, 384), *ref["dW"])


def test_fuse_head_split_text_stage_equals_one_launch():
    """the benchmarked split path: a text-stage launch (no W) writes text_feature, the final launch takes it as tf_in;
    same masks, same bits as the single launch"""
    h = _Head(32, 128, 256, 6, False, False, seed=11)
    rc, one = h.run(True, 0.3, 99, 5)
    _, text = h.run(True, 0.3, 99, 5, loss=False)
    rc2, split = h.run(True, 0.3, 99, 5, tf_in=text["tf"].to(DEV))
    for k in ("af", "out", "loss", "dw", "W", "m", "v"):
        assert torch.equal(one[k], split[k]), k
    assert torch.equal(one["tf"], text["tf"])


def test_fuse_head_rejects_one_past_the_shared_memory_limit():
    """T up to the 200 KB of one CTA runs; one more time step returns UNSUPPORTED (and launches nothing)"""
    Ht, Ha = 128, 256
    F = Ht + Ha

    def fits(T):
        return (3 * Ht + 2 * F + Ha + ((T + 3) & ~3) + T * Ht + 32) * 4 <= 200 * 1024

    T = max(t for t in range(1, 1000) if fits(t))
    h = _Head(2, Ht, Ha, T, False, False, seed=2)
    rc, r = h.run(False, 0.0, 1, 0)
    L, _ = _lib()
    L.check(rc, "fuse_head at the limit")
    ctx_ref, S = sh.attention_pool(h.seq, h.h_n, h.w_att, h.b_att)
    _check(f"fuse_head/Tmax{T}", "ctx_out", r["ctx"], ctx_ref, S)
    h2 = _Head(2, Ht, Ha, T + 1, False, False, seed=2)
    rc, _ = h2.run(False, 0.0, 1, 0)
    assert rc != 0 and "too large" in L.load().b200rnn_last_error().decode()


def test_fuse_head_adam_is_bit_identical_to_adamw():
    """one Adam rule: the in-kernel update and b200rnn_adamw (the all-reduce path) from the same dW"""
    for t0 in (0, 1, 4, 999):
        h = _Head(40, 128, 256, 0, False, False, seed=t0 + 1)
        _, r = h.run(True, 0.3, 3, 7, t0=t0)
        C, F = 2, 384
        P = h.dev["W"].clone().view(-1)
        M = _d(np.full(C * F, 1e-3, np.float32))
        V = _d(np.full(C * F, 1e-6, np.float32))
        step = torch.tensor(float(t0), device=DEV)
        _adamw(P, r["dw"][:C * F].to(DEV), M, V, step, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1.0)
        torch.cuda.synchronize()
        assert torch.equal(P.cpu(), r["W"].view(-1)) and torch.equal(M.cpu(), r["m"]) and torch.equal(V.cpu(), r["v"])
        assert r["step"].item() == step.item() == t0 + 1


# ---- inter-layer dropout of GRU / LSTM (dropout_kernel) ------------------------------------------------------------------
@pytest.mark.parametrize("mode,H,bidir,ragged,proj,grad", [
    ("gru", 256, False, False, 0, False), ("lstm", 128, True, False, 0, False), ("gru", 64, True, False, 0, True),
    ("lstm", 128, False, True, 0, True), ("gru", 256, True, False, 0, True), ("lstm", 128, True, False, 32, True)])
def test_inter_layer_dropout_masks_are_the_oracles(mode, H, bidir, ragged, proj, grad):
    """L = 3, p = 0.3: the module's output (and with `grad` its BPTT: dx and every weight gradient) equals per-layer
    float64 torch modules with the masks of oracle.philox (stream = layer index, element (t B + b) D W + j of the layer
    output of width W = H or proj_size, offset from _rng_state), normwise at the fp32 recurrence's level; a mask read
    from the wrong word, stream or offset is an O(1) error. The offset advances by ceil(T B D W / 4) per forward, and
    a second forward draws the masks of the advanced offset."""
    import b200rnn

    torch.manual_seed(0)
    T, B, I, L_, p = 9, 5 if not ragged else 6, 48, 3, 0.3
    cls = torch.nn.GRU if mode == "gru" else torch.nn.LSTM
    kw = dict(proj_size=proj) if proj else {}
    ref = cls(I, H, num_layers=L_, bidirectional=bidir, dropout=p, **kw)
    mine = b200rnn.from_torch(ref).to(DEV).train()
    D = 2 if bidir else 1
    W = proj or H
    n = T * B * D * W
    seed, off = 0xC0FFEE, 4242
    mine._rng_state.copy_(torch.tensor([seed, off], dtype=torch.int64))
    x = torch.randn(T, B, I)
    wy = torch.randn(T, B, D * W)
    lengths = torch.tensor([9, 9, 7, 4, 2, 1]) if ragged else None
    per = [cls(I if l == 0 else D * W, H, bidirectional=bidir, **kw).double() for l in range(L_)]
    for l, m in enumerate(per):
        for name, prm in m.named_parameters():
            prm.data.copy_(getattr(ref, name.replace("_l0", f"_l{l}")).data.double())
    for rep in range(2):
        o = off + rep * ((n + 3) // 4)
        xd = x.to(DEV).requires_grad_(grad)
        mine.zero_grad(set_to_none=True)
        with torch.set_grad_enabled(grad):
            if ragged:
                packed = torch.nn.utils.rnn.pack_padded_sequence(xd, lengths, enforce_sorted=False)
                y = torch.nn.utils.rnn.pad_packed_sequence(mine(packed)[0], total_length=T)[0]
            else:
                y = mine(xd)[0]
            if grad:
                (y * wy.to(DEV)).sum().backward()
        torch.cuda.synchronize()
        assert mine._rng_state[1].item() == o + (n + 3) // 4
        for m in per:
            m.zero_grad(set_to_none=True)
        x64 = x.double().requires_grad_(grad)
        h = x64
        for l, m in enumerate(per):
            if ragged:
                h = torch.nn.utils.rnn.pad_packed_sequence(
                    m(torch.nn.utils.rnn.pack_padded_sequence(h, lengths, enforce_sorted=False))[0], total_length=T)[0]
            else:
                h = m(h)[0]
            if l < L_ - 1:
                f = philox.dropout_factor(seed, o, l, n, p).reshape(T, B, D * W)
                h = h * torch.from_numpy(f).double()
        tag = f"inter_layer_dropout/{mode}{H}{f'-proj{proj}' if proj else ''}-D{D}-{'ragged' if ragged else 'dense'}"
        err = ((y.detach().double().cpu() - h.detach()).norm() / h.detach().norm()).item()
        RESULTS[f"{tag}/y_rel_err_rep{rep}"] = err
        assert err < 1e-5, err
        if grad:
            (h * wy.double()).sum().backward()
            pairs = [(xd.grad, x64.grad, "dx")]
            for l, m in enumerate(per):
                for name, prm in m.named_parameters():
                    pairs.append((getattr(mine, name.replace("_l0", f"_l{l}")).grad, prm.grad, name + f"@{l}"))
            for got, want, name in pairs:
                e = ((got.double().cpu() - want).norm() / want.norm()).item()
                RESULTS[f"{tag}/d{name}_rel_err_rep{rep}"] = max(RESULTS.get(f"{tag}/d{name}_rel_err_rep{rep}", 0), e)
                assert e < 1e-4, (name, e)


def test_inter_layer_dropout_cuda_graph_replays_draw_advanced_offsets():
    """a captured module forward: every replay reads {seed, offset} from the device state and advances it, so replay k
    draws the masks of offset + k ceil(T B D H / 4)"""
    import b200rnn

    torch.manual_seed(1)
    T, B, I, H, L_, p = 7, 4, 32, 64, 2, 0.3
    ref = torch.nn.GRU(I, H, num_layers=L_, dropout=p)
    mine = b200rnn.from_torch(ref).to(DEV).train()
    x = torch.randn(T, B, I, device=DEV)
    consume = (T * B * H + 3) // 4
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                mine(x)
        torch.cuda.current_stream().wait_stream(s)
        seed, off = 0xABCDEF, 1000
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y = mine(x)[0]
        mine._rng_state.copy_(torch.tensor([seed, off], dtype=torch.int64))
        per = [torch.nn.GRU(I if l == 0 else H, H).double() for l in range(L_)]
        for l, m in enumerate(per):
            for name, prm in m.named_parameters():
                prm.data.copy_(getattr(ref, name.replace("_l0", f"_l{l}")).data.double())
        for k in range(3):
            graph.replay()
            torch.cuda.synchronize()
            assert mine._rng_state[1].item() == off + (k + 1) * consume
            h = per[0](x.double().cpu())[0]
            h = h * torch.from_numpy(philox.dropout_factor(seed, off + k * consume, 0, T * B * H, p).reshape(T, B, H)).double()
            h = per[1](h)[0]
            err = ((y.double().cpu() - h).norm() / h.norm()).item()
            assert err < 1e-5, (k, err)


# ---- LayerNorm prologue (layernorm_kernel / layernorm_bwd_kernel through b200rnn_debug_layernorm) --------------------------
LNB_BLOCKS = 2 * NUM_SMS


def _layernorm(x_t, rows, R, Cc, gamma, beta, eps, dy=None, dx=True, dgamma0=None, lengths=None, B=1):
    L, lib = _lib()
    fn = lib.b200rnn_debug_layernorm
    import ctypes

    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                   ctypes.c_int, ctypes.c_void_p]
    G, Bt = _d(gamma), _d(beta)
    out = torch.full((R, Cc), float("nan"), device=DEV)
    res = dict(y=out)
    args = dict(dy=None, dx=None, dg=None, db=None, part=None)
    if dy is not None:
        DY = _d(dy)
        dxt = torch.full_like(x_t, float("nan")) if dx else None
        dg = _d(dgamma0[0]) if dgamma0 is not None else torch.full((Cc,), float("nan"), device=DEV)
        db = _d(dgamma0[1]) if dgamma0 is not None else torch.full((Cc,), float("nan"), device=DEV)
        part = torch.empty(LNB_BLOCKS * 2 * Cc, device=DEV)
        args = dict(dy=DY, dx=dxt, dg=dg, db=db, part=part)
        res.update(dx=dxt, dgamma=dg, dbeta=db)
    LEN = _d(lengths.astype(np.int32)) if lengths is not None else None
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    L.check(fn(x_t.data_ptr(), rows[0], rows[1], rows[2], R, Cc, G.data_ptr(), Bt.data_ptr(), eps, out.data_ptr(),
               ptr(args["dy"]), ptr(args["dx"]), ptr(args["dg"]), ptr(args["db"]), int(dgamma0 is not None),
               ptr(args["part"]), LNB_BLOCKS * 2 * Cc, ptr(LEN), B, _stream()), "debug_layernorm")
    torch.cuda.synchronize()
    return {k: v.cpu() if v is not None else None for k, v in res.items()}


@pytest.mark.parametrize("Cc", [128, 256, 512, 1024])
@pytest.mark.parametrize("R", [1, 13, 8 * LNB_BLOCKS + 37])
@pytest.mark.parametrize("regime", ["normal", "offset1e3", "var_eps", "constant"])
def test_layernorm_fwd_bwd_within_bound(Cc, R, regime):
    """strided rows (time-major [T, B, ld], ld > Cc), ragged lengths, accumulate into dgamma / dbeta"""
    rng = np.random.default_rng(Cc + R)
    Bn = 3 if R > 1 else 1
    T = -(-R // Bn)
    ld = Cc + 12
    x = rng.standard_normal((T * Bn, Cc))
    if regime == "offset1e3":
        x = x + 1e3
    elif regime == "var_eps":
        x = x * math.sqrt(1e-5) + 0.5
    elif regime == "constant":
        x = np.repeat(rng.standard_normal((T * Bn, 1)), Cc, 1)
    x = x[:R].astype(np.float32)
    big = np.zeros((T, Bn, ld), np.float32)
    big.reshape(T * Bn, ld)[:R, :Cc] = x
    X = _d(big)
    rows = (Bn * ld, ld, Bn)
    gamma = rng.standard_normal(Cc).astype(np.float32)
    beta = rng.standard_normal(Cc).astype(np.float32)
    dy = rng.standard_normal((R, Cc)).astype(np.float32)
    eps = 1e-5
    lengths = None
    if R > 1:
        lengths = np.array([T, T - 1, max(T // 2, 0)][:Bn])
    old = (rng.standard_normal(Cc).astype(np.float32), rng.standard_normal(Cc).astype(np.float32))
    outs = [_layernorm(X, rows, R, Cc, gamma, beta, eps, dy=dy, dgamma0=old, lengths=lengths, B=Bn) for _ in range(2)]
    for k in outs[0]:
        assert torch.equal(outs[0][k].nan_to_num(7.0), outs[1][k].nan_to_num(7.0)), k
    live = np.ones(R, bool)
    if lengths is not None:
        r = np.arange(R)
        live = (r // Bn) < lengths[r % Bn]
    blocks = min((R + 7) // 8, LNB_BLOCKS)
    ref = sh.layernorm_bounds(x, gamma, beta, np.float32(eps), dy * live[:, None], nblocks=blocks)
    case = f"layernorm/Cc{Cc}-R{R}-{regime}"
    y, Sy = ref["y"]
    _check(case, "y", outs[0]["y"], np.where(live[:, None], y, 0.0), np.where(live[:, None], Sy, 0.0))
    dxk = outs[0]["dx"].reshape(T * Bn, ld)[:R]
    assert torch.isnan(outs[0]["dx"].reshape(T * Bn, ld)[:, Cc:]).all(), "dx writes only the row's Cc columns"
    dx, Sdx = ref["dx"]
    _check(case, "dx", dxk[:, :Cc], np.where(live[:, None], dx, 0.0), np.where(live[:, None], Sdx, 0.0))
    for name, o in (("dgamma", old[0]), ("dbeta", old[1])):
        v, S = ref[name]
        _check(case, name, outs[0][name], v + o, S + np.abs(v + o) + np.abs(o))


def test_layernorm_backward_without_dx_and_overwrite():
    """dx = NULL (only dgamma / dbeta), accumulate = 0 overwrites whatever the outputs held"""
    rng = np.random.default_rng(9)
    R, Cc = 40, 256
    x = rng.standard_normal((R, Cc)).astype(np.float32)
    gamma, beta = rng.standard_normal(Cc).astype(np.float32), rng.standard_normal(Cc).astype(np.float32)
    dy = rng.standard_normal((R, Cc)).astype(np.float32)
    o = _layernorm(_d(x), (0, Cc, 1 << 30), R, Cc, gamma, beta, 1e-5, dy=dy, dx=False)
    ref = sh.layernorm_bounds(x, gamma, beta, np.float32(1e-5), dy, nblocks=5)
    _check("layernorm/no_dx", "dgamma", o["dgamma"], *ref["dgamma"])
    _check("layernorm/no_dx", "dbeta", o["dbeta"], *ref["dbeta"])


# ---- dropout_kernel directly: the float4 path and the scalar tail --------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 4, 4097, 1 << 20])
@pytest.mark.parametrize("shift", [0, 1, 2])
@pytest.mark.parametrize("p", [0.3, 0.5, 1.0])
def test_dropout_kernel_mask_exact(n, shift, p):
    """in and out shifted by `shift` floats from a 16-byte boundary: shift 0 takes the float4 path for every whole
    quad, any other shift the scalar path; n % 4 != 0 ends in a partial quad. Every output is in * factor exactly."""
    import ctypes

    L, lib = _lib()
    lib.b200rnn_debug_dropout.restype = ctypes.c_int
    lib.b200rnn_debug_dropout.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_float,
                                          ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p,
                                          ctypes.c_void_p]
    rng = np.random.default_rng(n + shift)
    x = rng.standard_normal(n + 8).astype(np.float32)
    X = _d(x)
    Y = torch.full((n + 8,), float("nan"), device=DEV)
    hdr = torch.zeros(2, dtype=torch.int64, device=DEV)
    seed, off, stream = 0xDEADBEEF12345, 77777, 2
    L.check(lib.b200rnn_debug_dropout(X.data_ptr() + 4 * shift, Y.data_ptr() + 4 * shift, n, p, seed, off, stream,
                                      hdr.data_ptr(), _stream()), "debug_dropout")
    torch.cuda.synchronize()
    y = Y.cpu().numpy()
    f = philox.dropout_factor(seed, off, stream, n, p)
    want = (x[shift:shift + n] * f).astype(np.float32)
    assert np.array_equal(y[shift:shift + n], want)
    assert np.isnan(y[:shift]).all() and np.isnan(y[shift + n:]).all(), "nothing outside [0, n) is written"


# ---- the benchmarked step, in the mode it is benchmarked in ------------------------------------------------------------------
def test_fused_fuse_step_train_mode_vs_float64_composition():
    """FusedFuseStep on bench.py's FUSE_ARGS model (dropout 0.3, train mode, the split text stage) for three steps,
    against float64: the masked encoder oracle (oracle.rnn_numpy with every inter-layer mask of oracle.philox, at the
    offsets read from the modules' device states), LayerNorm, attention pooling, both heads with the head's four
    streams, the loss and Adam. Features, probabilities, loss, d fc_final.0.weight and the weight, normwise. The
    device offsets advance by ceil(T B D H / 4) per encoder and by FusedFuseStep's rng_consume per step."""
    import b200rnn
    from oracle.rnn_numpy import NumpyRNN

    args = dict(text_embed_size=1024, text_hidden_dims=128, rnn_layers=2, dropout=0.3, num_classes=2,
                audio_hidden_dims=256, audio_embed_size=256)
    torch.manual_seed(0)
    m = b200rnn.fusion_net(**args).to(DEV)
    for prm in m.parameters():
        prm.requires_grad = False
    m.fc_final[0].weight.requires_grad = True
    m.train()
    lr = 1e-3
    step = b200rnn.FusedFuseStep(m, lr=lr)
    B, Ta, Tt = 4, 120, 30
    f64 = lambda t: t.detach().double().cpu().numpy()  # noqa: E731
    txt = NumpyRNN("lstm", [f64(q) for q in m.lstm_net.parameters()], 2, True)
    aud = NumpyRNN("gru", [f64(q) for q in m.lstm_net_audio.parameters()], 2, False)
    W = f64(m.fc_final[0].weight).astype(np.float32)
    mom, vel = np.zeros(W.size, np.float32), np.zeros(W.size, np.float32)
    g = torch.Generator().manual_seed(3)
    for it in range(3):
        audio, text = torch.randn(B, Ta, 256, generator=g), torch.randn(B, Tt, 1024, generator=g)
        y = torch.randint(0, 2, (B,), generator=g)
        st_t, st_a, st_h = (m.lstm_net._rng_state.cpu().tolist(), m.lstm_net_audio._rng_state.cpu().tolist(),
                            step.rng_state.cpu().tolist())
        probs, loss = step(b200rnn.FuseBatch(audio.to(DEV), text.to(DEV)), y.to(DEV))
        torch.cuda.synchronize()
        consume = (B * 256 + 3) // 4
        assert m.lstm_net._rng_state[1].item() == st_t[1] + (Tt * B * 256 + 3) // 4
        assert m.lstm_net_audio._rng_state[1].item() == st_a[1] + (Ta * B * 256 + 3) // 4
        assert step.rng_state[1].item() == st_h[1] + consume
        # float64 composition
        mt = [philox.dropout_factor(st_t[0], st_t[1], 0, Tt * B * 256, 0.3).reshape(Tt, B, 256)]
        seq, h_n, _ = txt.forward(text.double().numpy().transpose(1, 0, 2), masks=mt)
        ma = [philox.dropout_factor(st_a[0], st_a[1], 0, Ta * B * 256, 0.3).reshape(Ta, B, 256)]
        xa, _, _ = sh.layernorm(audio.double().numpy().transpose(1, 0, 2), f64(m.ln.weight), f64(m.ln.bias), m.ln.eps)
        ya, _ = aud.forward(xa, masks=ma)
        pooled = ya.sum(0)
        ctx, _ = sh.attention_pool(seq, h_n, f64(m.attention_layer[0].weight), f64(m.attention_layer[0].bias))
        fac = lambda s_, n_: philox.dropout_factor(st_h[0], st_h[1], s_, B * n_, 0.3).reshape(B, n_)  # noqa: E731
        tf, _, _ = sh.mlp_dropout(ctx, f64(m.fc_out[1].weight), f64(m.fc_out[1].bias), fac(0, 128), fac(1, 128), 1)
        af, _, _ = sh.mlp_dropout(pooled, f64(m.fc_audio[1].weight), f64(m.fc_audio[1].bias), fac(2, 256), fac(3, 256), 1)
        r = sh.fuse_head_loss(tf, af, W, y.numpy())
        a = sh.adam(W.reshape(-1), r["dW"][0].reshape(-1).astype(np.float32), mom, vel, it + 1, np.float32(lr),
                    np.float32(0.9), np.float32(0.999), np.float32(1e-8))
        W_new = a["p"][0]

        def rel(got, want):
            got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
            return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))

        errs = dict(probs=rel(f64(probs), r["out"][0]), loss=rel(loss.item(), r["loss"][0]),
                    dw=rel(f64(step.dw)[:768], r["dW"][0].reshape(-1)),
                    update=rel(f64(m.fc_final[0].weight).reshape(-1) - W.reshape(-1), W_new - W.reshape(-1)))
        for k, v in errs.items():
            RESULTS[f"fused_fuse_step_train/step{it}/{k}_rel_err"] = v
        assert errs["probs"] < 1e-4 and errs["loss"] < 1e-4 and errs["dw"] < 1e-3, errs
        assert errs["update"] < 1e-3, errs
        W = f64(m.fc_final[0].weight).astype(np.float32)
        mom, vel = f64(step.m).astype(np.float32), f64(step.v).astype(np.float32)
