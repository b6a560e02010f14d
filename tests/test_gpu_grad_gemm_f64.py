"""Every mode of the backward's gradient GEMMs against float64, element by element.

The backward hands each gradient GEMM (dW_ih, the shifted dW_hh, the h_0 term, dW_hr, dX) to run_grad_gemm
(csrc/api.cu), which runs it on the tensor cores (tc_gemm_presplit: TF32 split once per source, MN-major operands read
by the kernel's own loads, split-K over the persistent CTAs and a fixed-order reduce) or on the FFMA GEMM. The test-only
entry b200rnn_debug_grad_gemm runs that same function on sources and GEMMs given here, so every mode is reached
directly: both paths, the (MN, MN) wgrad and (K, MN) dgrad layouts (all four on FFMA), row offsets (row0 = B), split-K
with K tails and short last splits, accumulate, single-pass TF32, strided outputs, and sources shared between GEMMs.

Oracle: the float64 product of the fp32 operands as the GEMM addresses them (row map, row0), plus C0 when accumulating;
in TF32 mode the operands are rounded to TF32 first (oracle.tf32.round_tf32), so only the accumulation error is left.

Bound, per element: |C - C64| <= kappa u S with S = (|A| |B|)_ij (+ |C0_ij|), u = 2^-24 in both modes and

    kappa = 3 (sqrt(chain) + sqrt(splitk)) + 1  [+ 48 + 20 on 3xTF32 tensor cores, + 16 on TF32 ones]

chain = k-blocks per split (tensor cores) or K values per split (FFMA), splitk = the split count the launch ran with
(both returned by the entry). The stages, counted as in tests/test_gpu_numerics_f64.py (derivation in
oracle/grad_gemm.py): 20u per product for the 3xTF32 split (the dropped lo*lo and the TF32 reading of both lo
operands, worst case); 4u per MMA for the truncating accumulation inside a k-block (12 MMAs in 3xTF32, 4 in TF32,
counted linearly because truncation is biased); the round-to-nearest chains over k-blocks (or fmaf over K) and over
splits, each sqrt(depth) u S with high probability (Higham & Mary 2019), taken 3 times because the maximum runs over
up to 10^7 elements; one rounding for C0. tests/test_grad_gemm_bound_cpu.py checks the bound on a numpy emulation.

Sharp operands: positive a = h (1 + 2^-12) with h exactly TF32, so hi = h and lo = 2^-12 h exactly; a lost correction
product then shifts every output by 2^-12 S = 4096 u S, and rows of A / columns of B scaled by 2^e, e in [-20, 20],
make the small outputs count on their own. Sentinels: NaN in every source row and column no GEMM addresses, C filled
with NaN before a GEMM that does not accumulate, a fixed bit pattern in C's padding columns and in the rows past M;
all must come out as they went in. Every GEMM is run twice and must be bitwise repeatable, and one with a row offset
must equal, bit for bit, the same GEMM on a copy of its operand that starts at row 0.

Coverage: real backwards (GRU and BiLSTM at the project's shapes, D = 1 and 2, hx, ragged, fused LayerNorm, a
misaligned gradient sink, a frozen weight_ih_l0, TF32) run with B200RNN_DEBUG, which prints one line per gradient GEMM;
every mode tuple they produce must also be produced by this file's matrix, read from the matrix's own debug lines.

B200RNN_NUMERICS_RECORD=<path> writes the max err / bound per case as JSON."""
import ctypes
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from oracle.grad_gemm import U, kappa

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
SENTINEL = 0x7FC0BEEF   # C's padding: a NaN payload no arithmetic produces
LINEAR = 0x7FFFFFFF     # inner_n of a dense row map
RECORDS = {}


@pytest.fixture(scope="module", autouse=True)
def _record():
    yield
    path = os.environ.get("B200RNN_NUMERICS_RECORD")
    if path and RECORDS:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip().splitlines()
        largest = max(RECORDS, key=RECORDS.get)
        with open(path, "w") as f:
            json.dump({"device": q[0] if q else "unknown", "largest": [largest, RECORDS[largest]],
                       "max_err_over_bound": RECORDS}, f, indent=1, sort_keys=True)
            f.write("\n")


# ---- the entry --------------------------------------------------------------------------------------------------------

def _entry():
    from b200rnn import _lib

    fn = _lib.load().b200rnn_debug_grad_gemm
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                   ctypes.POINTER(ctypes.c_size_t), ctypes.c_void_p, ctypes.c_void_p]
    return fn


def _rows_off(rows, R):
    s_outer, s_inner, inner_n = rows
    r = torch.arange(R, device=DEV, dtype=torch.int64)
    return (r // inner_n) * s_outer + (r % inner_n) * s_inner


class Src:
    """an fp32 source [R][C]: `vals` (NaN wherever no GEMM reads) laid out in a NaN-filled buffer through a row map,
    dense (row stride C + pad) or batch-first [tb][R / tb][ld] (rows r = t * tb + b)"""

    def __init__(self, vals, tb=None, pad=4):
        self.vals = vals
        R, C = vals.shape
        ld = C + pad
        self.rows = (0, ld, LINEAR) if tb is None else (ld, (R // tb) * ld, tb)
        self.buf = torch.full((R * ld + pad,), float("nan"), device=DEV)
        idx = _rows_off(self.rows, R)[:, None] + torch.arange(C, device=DEV)[None, :]
        self.buf[idx.reshape(-1)] = vals.reshape(-1)

    def desc(self):
        return [self.buf.data_ptr(), *self.rows, *self.vals.shape]

    def operand(self, row0, kcontig, mn, K):
        """the operand as a GEMM addresses it: A [mn][K] (kcontig) or [K][mn], returned as [mn][K]"""
        v = self.vals[row0:row0 + (mn if kcontig else K)]
        return v[:, :K] if kcontig else v[:, :mn].t()


class Out:
    """C [M][N] in a buffer of sentinels: dense (row stride N + pad) or batch-first (rows m = t * tb + b)"""

    def __init__(self, M, N, tb=None, C0=None):
        ld = (N + 3) // 4 * 4 + 4
        self.M, self.N = M, N
        self.rows = (0, ld, LINEAR) if tb is None else (ld, (M // tb) * ld, tb)
        self.buf = torch.full(((M + 1) * ld,), 0, dtype=torch.int32, device=DEV).fill_(SENTINEL).view(torch.float32)
        self.idx = (_rows_off(self.rows, M)[:, None] + torch.arange(N, device=DEV)[None, :]).reshape(-1)
        self.C0 = C0
        self.buf[self.idx] = float("nan") if C0 is None else C0.reshape(-1)
        self.init = self.buf.clone()

    def value(self):
        return self.buf[self.idx].view(self.M, self.N)

    def outside_untouched(self):
        mask = torch.ones_like(self.buf, dtype=torch.bool)
        mask[self.idx] = False
        return torch.equal(self.buf.view(torch.int32)[mask], self.init.view(torch.int32)[mask])


def _run(srcs, gemms, tf32):
    """run `gemms` [(a, b, M, N, K, out, accumulate, splitk, tc)], a = (src, row0, kcontig), in order through one call;
    returns the (splitk, chunk) each ran with"""
    fn = _entry()
    sidx = {id(s): i for i, s in enumerate(srcs)}
    s_arr = torch.tensor([v for s in srcs for v in s.desc()], dtype=torch.int64)
    g_rows = []
    for (a, b, M, N, K, out, acc, splitk, tc) in gemms:
        g_rows.append([sidx[id(a[0])], a[1], int(a[2]), sidx[id(b[0])], b[1], int(b[2]), M, N, K, out.buf.data_ptr(),
                       *out.rows, int(acc), int(splitk), int(tc)])
    g_arr = torch.tensor(g_rows, dtype=torch.int64)
    plans = torch.zeros(2 * len(gemms), dtype=torch.int32)
    need = ctypes.c_size_t(0)
    st = torch.cuda.current_stream(DEV).cuda_stream
    from b200rnn import _lib

    _lib.check(fn(s_arr.data_ptr(), len(srcs), g_arr.data_ptr(), len(gemms), int(tf32), None, ctypes.byref(need),
                  None, st), "b200rnn_debug_grad_gemm")
    scratch = torch.empty(need.value, dtype=torch.uint8, device=DEV)
    _lib.check(fn(s_arr.data_ptr(), len(srcs), g_arr.data_ptr(), len(gemms), int(tf32), scratch.data_ptr(),
                  ctypes.byref(need), plans.data_ptr(), st), "b200rnn_debug_grad_gemm")
    torch.cuda.synchronize()
    return [tuple(plans[2 * j:2 * j + 2].tolist()) for j in range(len(gemms))]


def _rtf32(x):
    """cvt.rna.tf32.f32 of float32 x (oracle.tf32.round_tf32, on the device)"""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & -8192).view(torch.float32)


def _check(name, gemm, plan, tf32):
    (a, b, M, N, K, out, acc, _, tc) = gemm
    A = a[0].operand(a[1], a[2], M, K).double()
    B = b[0].operand(b[1], b[2], N, K).double().t()
    if tc and tf32:
        A, B = _rtf32(A).double(), _rtf32(B).double()
    assert not (torch.isnan(A).any() or torch.isnan(B).any()), "a sentinel sits inside the addressed operand"
    C64 = A @ B
    S = A.abs() @ B.abs()
    if acc:
        C64 = C64 + out.C0.double()
        S = S + out.C0.double().abs()
    C = out.value()
    assert torch.isfinite(C).all(), (name, "non-finite output: a sentinel was read or C was not written")
    assert out.outside_untouched(), (name, "a padding column or a row past M was written")
    splitk, chunk = plan
    nkb = (K + 31) // 32
    chain = min(chunk, nkb) if tc else min(chunk, K)
    kap = kappa("tc" if tc else "ffma", tf32 and tc, chain, splitk)
    ratio = ((C.double() - C64).abs() / (kap * U * S)).max().item()
    RECORDS[name] = max(RECORDS.get(name, 0.0), ratio)
    assert ratio <= 1.0, (name, ratio, kap, plan)


def _program(prog, tf32, check=True, name="case"):
    """prog() -> (srcs, gemms); runs it twice (bitwise repeatable) and checks every GEMM against float64"""
    srcs, gemms = prog()
    plans = _run(srcs, gemms, tf32)
    if not check:
        return
    first = [g[5].buf.clone() for g in gemms]
    for g in gemms:   # same inputs again: C0 restored, or NaN
        g[5].buf.copy_(g[5].init)
    assert _run(srcs, gemms, tf32) == plans
    for j, g in enumerate(gemms):
        assert torch.equal(g[5].buf.view(torch.int32), first[j].view(torch.int32)), (name, j, "not repeatable")
        _check("%s/%d" % (name, j), g, plans[j], tf32)
    return srcs, gemms, plans


# ---- operands ---------------------------------------------------------------------------------------------------------

def _gen(seed):
    return torch.Generator(DEV).manual_seed(seed)


def _sharp(shape, g, scale_dim):
    h = _rtf32(1.0 + torch.rand(shape, device=DEV, generator=g))
    e = torch.randint(-20, 21, (shape[0], 1) if scale_dim == 0 else (1, shape[1]), device=DEV, generator=g)
    return h * (1.0 + 2.0 ** -12) * torch.exp2(e.float()), e


def _operands(M, N, K, data, seed):
    """A_eff [M][K], B_eff [K][N] and a C0 of the outputs' magnitude"""
    g = _gen(seed)
    if data == "sharp":
        A, ea = _sharp((M, K), g, 0)
        B, eb = _sharp((K, N), g, 1)
        scale = torch.exp2((ea + eb).float())
    else:
        A = torch.randn(M, K, device=DEV, generator=g)
        B = torch.randn(K, N, device=DEV, generator=g)
        scale = 1.0
    C0 = torch.randn(M, N, device=DEV, generator=g) * math.sqrt(K) * scale
    return A, B, C0


def _place(op, row0, kcontig, tc, tb=None, extra_rows=1):
    """a source holding operand op [mn][K] at row0 in the layout the GEMM reads, NaN everywhere else (rows before row0
    and past the operand, columns past its width up to the source's width, padding up to the row stride)"""
    body = op if kcontig else op.t()
    R = row0 + body.shape[0] + (tb if tb else extra_rows)
    C = body.shape[1] + 1
    if tc:
        C = (C + 3) // 4 * 4
    vals = torch.full((R, C), float("nan"), device=DEV)
    vals[row0:row0 + body.shape[0], :body.shape[1]] = body
    return Src(vals, tb=tb)


# ---- the matrix -------------------------------------------------------------------------------------------------------

def _single(path, a_kc, b_kc, M, N, K, row0=(0, 0), acc=0, splitk=True, data="sharp", seed=0, copy_rows=False):
    tc = path == "tc"

    def prog():
        A, B, C0 = _operands(M, N, K, data, seed)
        r0 = (0, 0) if copy_rows else row0
        sa = _place(A, r0[0], a_kc, tc)
        sb = _place(B.t(), r0[1], b_kc, tc)
        out = Out(M, N, C0=C0 if acc else None)
        return [sa, sb], [((sa, r0[0], a_kc), (sb, r0[1], b_kc), M, N, K, out, acc, splitk, tc)]
    return prog


def _lay(kc):
    return "k" if kc else "mn"


GENERIC = {}
ROW0 = {}   # the row-offset cases: (args, kwargs) of _single
for _path in ("tc", "ffma"):
    _layouts = [(False, False), (True, False)] + ([(True, True), (False, True)] if _path == "ffma" else [])
    _N = 128 if _path == "tc" else 130
    for _akc, _bkc in _layouts:
        for _K in (1, 31, 32, 33, 1100):
            for _acc in (0, 1):
                for _tf32 in ((False, True) if _path == "tc" else (False,)):
                    GENERIC["%s_%s%s_K%d_acc%d%s" % (_path, _lay(_akc), _lay(_bkc), _K, _acc, "_tf32" * _tf32)] = (
                        _single(_path, _akc, _bkc, 129, _N, _K, acc=_acc), _tf32)
        # row offsets of the MN-major operands (the shifted dW_hh: row0 = B on one side)
        for _K in (33, 1100):
            for _r0 in ((64, 0), (0, 64)):
                if _akc and _r0[0]:
                    continue
                for _acc in (0, 1):
                    _name = "%s_%s%s_K%d_row0_%d_%d_acc%d" % (_path, _lay(_akc), _lay(_bkc), _K, _r0[0], _r0[1], _acc)
                    ROW0[_name] = ((_path, _akc, _bkc, 129, _N, _K), {"row0": _r0, "acc": _acc})
                    GENERIC[_name] = (_single(*ROW0[_name][0], **ROW0[_name][1]), False)
    # split-K off, and M / N at the tile sizes (odd N on FFMA)
    GENERIC["%s_mnmn_K1100_nosplit" % _path] = (_single(_path, False, False, 129, _N, 1100, splitk=False), False)
    GENERIC["%s_mnmn_K1100_nosplit_acc1" % _path] = (_single(_path, False, False, 129, _N, 1100, acc=1, splitk=False),
                                                    False)
    _mns = [(1, 128), (256, 256), (384, 1024), (512, 256), (768, 128), (1024, 1024)]
    if _path == "ffma":
        _mns += [(129, 200), (300, 37)]
    for _M, _NN in _mns:
        GENERIC["%s_mnmn_M%d_N%d_K1100" % (_path, _M, _NN)] = (_single(_path, False, False, _M, _NN, 1100, acc=1), False)
# random operands at small K: there a lost product is large against the bound even with random signs
for _K in (1, 31, 32, 33):
    GENERIC["tc_mnmn_K%d_random" % _K] = (_single("tc", False, False, 129, 128, _K, data="random", seed=1), False)
    GENERIC["tc_kmn_K%d_random" % _K] = (_single("tc", True, False, 129, 128, _K, data="random", seed=2), False)


# The project's backward shapes (I, H, B, T, gates): the c2 / audio GRU-256 and the text BiLSTM (H = 128, I = 1024)
FAMILIES = {
    "c2_gru": (256, 256, 64, 120, 3),
    "audio_gru": (256, 256, 128, 120, 3),
    "text_lstm_b64": (1024, 128, 64, 30, 4),
    "text_lstm_b128": (1024, 128, 128, 30, 4),
}


def _family_progs(fam):
    """the backward's GEMMs of one layer at a family's shape, sharing their sources as the backward does:
    dW_ih then dX on one dG split; the shifted dW_hh (GRU: r,z from dG, then n from dn*r on the same h split) in both
    directions; the h_0 term. Batch-first x, y and dx (row maps of the caller's tensors)."""
    I, H, B, T, G = FAMILIES[fam]
    GH, TB, Kp = G * H, T * B, (T - 1) * B
    progs = {}
    for path, tf32s in (("tc", (False, True)), ("ffma", (False,))):
        tc = path == "tc"
        for acc in (0, 1):
            for tf32 in tf32s:
                tag = "%s_%s_acc%d%s" % (fam, path, acc, "_tf32" * tf32)

                def ih(tc=tc, acc=acc):
                    g = _gen(11)
                    dG = torch.randn(TB, GH, device=DEV, generator=g)
                    X = torch.randn(TB, I, device=DEV, generator=g)
                    W = torch.randn(GH, I, device=DEV, generator=g) / math.sqrt(I)
                    sdg = Src(dG)
                    sx = _place(X.t(), 0, False, tc, tb=B)
                    sw = Src(W)
                    c0w = torch.randn(GH, I, device=DEV, generator=g) * math.sqrt(TB)
                    c0x = torch.randn(TB, I, device=DEV, generator=g) * math.sqrt(GH)
                    dw = Out(GH, I, C0=c0w if acc else None)
                    dx = Out(TB, I, tb=B, C0=c0x if acc else None)
                    return [sdg, sx, sw], [((sdg, 0, False), (sx, 0, False), GH, I, TB, dw, acc, True, tc),
                                           ((sdg, 0, True), (sw, 0, False), TB, I, GH, dx, acc, False, tc)]
                progs["%s_ih_dx" % tag] = (ih, tf32)
                for rev in (False, True):
                    g0, h0 = (0, B) if rev else (B, 0)

                    def hh(tc=tc, acc=acc, g0=g0, h0=h0):
                        g = _gen(12)
                        dG = torch.randn(TB, GH, device=DEV, generator=g)
                        h = torch.randn(TB, H, device=DEV, generator=g)
                        rz = 2 * H if G == 3 else GH
                        vals = torch.full((TB, GH + 4), float("nan"), device=DEV)
                        vals[g0:g0 + Kp, :rz] = dG[g0:g0 + Kp, :rz]   # nothing reads the n columns or the other rows
                        sdg = Src(vals)
                        hv = torch.full((TB, H), float("nan"), device=DEV)
                        hv[h0:h0 + Kp] = h[h0:h0 + Kp]
                        sh = Src(hv, tb=B)
                        c0 = torch.randn(GH, H, device=DEV, generator=g) * math.sqrt(Kp)
                        o1 = Out(rz, H, C0=c0[:rz] if acc else None)
                        gemms = [((sdg, g0, False), (sh, h0, False), rz, H, Kp, o1, acc, True, tc)]
                        srcs = [sdg, sh]
                        if G == 3:
                            dn = torch.full((TB, H + 4), float("nan"), device=DEV)
                            dn[g0:g0 + Kp, :H] = torch.randn(Kp, H, device=DEV, generator=g)
                            sdn = Src(dn)
                            o2 = Out(H, H, C0=c0[rz:] if acc else None)
                            gemms.append(((sdn, g0, False), (sh, h0, False), H, H, Kp, o2, acc, True, tc))
                            srcs.append(sdn)
                        return srcs, gemms
                    progs["%s_hh%s" % (tag, "_rev" if rev else "")] = (hh, tf32)

    def h0term():
        g = _gen(13)
        rows0 = Src(torch.randn(B, GH, device=DEV, generator=g))
        h0 = Src(torch.randn(B, H, device=DEV, generator=g))
        out = Out(GH, H, C0=torch.randn(GH, H, device=DEV, generator=g) * math.sqrt(B))
        return [rows0, h0], [((rows0, 0, False), (h0, 0, False), GH, H, B, out, 1, False, False)]
    progs["%s_h0" % fam] = (h0term, False)
    return progs


REAL = {}
for _fam in FAMILIES:
    REAL.update(_family_progs(_fam))


@pytest.mark.parametrize("name", list(GENERIC))
def test_grad_gemm_matrix_vs_f64(name):
    prog, tf32 = GENERIC[name]
    _program(prog, tf32, name=name)


@pytest.mark.parametrize("name", list(ROW0))
def test_row_offset_equals_a_copy_starting_at_row_0(name):
    """row0 = B reads the same numbers as a copy of the operand that starts at row 0, so C must be bit-identical"""
    args, kw = ROW0[name]
    shifted = _program(_single(*args, **kw), False, name=name)
    copied = _program(_single(*args, **kw, copy_rows=True), False, name=name + "/copy")
    assert shifted[2] == copied[2]
    assert torch.equal(shifted[1][0][5].value().view(torch.int32), copied[1][0][5].value().view(torch.int32))


@pytest.mark.parametrize("name", list(REAL))
def test_backward_shapes_vs_f64(name):
    prog, tf32 = REAL[name]
    _program(prog, tf32, name=name)


@pytest.mark.parametrize("data", ["sharp", "random"])
@pytest.mark.parametrize("M,N,K", [(1000, 384, 256), (3840, 512, 1024)])
def test_forward_projection_fp32_a_vs_f64(M, N, K, data):
    """the forward input projection's fp32-A kernel (A split in registers, its own MMA sequence issue_ra) under the same
    bound, one split of K / 32 k-blocks; its results equal the presplit kernel's (tests/test_gpu_gemm_f32a.py)"""
    from b200rnn import _lib

    fn = _lib.load().b200rnn_debug_gemm_f32a
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
                   ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                   ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    A, Bt, _ = _operands(M, N, K, data, seed=M + N)
    W = Bt.t().contiguous()
    A = A.contiguous()
    C = torch.full((M, N), float("nan"), device=DEV)
    bias = torch.zeros(N, device=DEV)
    sbytes = 8 * (M + N) * K + 4096
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=DEV)
    _lib.check(fn(M, N, K, A.data_ptr(), K, 0, 0, W.data_ptr(), C.data_ptr(), bias.data_ptr(), None, 0,
                  scratch.data_ptr(), sbytes, torch.cuda.current_stream(DEV).cuda_stream), "b200rnn_debug_gemm_f32a")
    torch.cuda.synchronize()
    A64, W64 = A.double(), W.double()
    C64, S = A64 @ W64.t(), A64.abs() @ W64.abs().t()
    ratio = ((C.double() - C64).abs() / (kappa("tc", False, K // 32, 1) * U * S)).max().item()
    RECORDS["fwd_f32a_M%d_N%d_K%d_%s" % (M, N, K, data)] = ratio
    assert ratio <= 1.0, ratio


# ---- coverage: every mode the backward runs is in the matrix --------------------------------------------------------

def _tuple(line):
    """the mode tuple of one '[b200rnn] grad gemm' line: path, layouts, row0 != 0, split-K, short last split, K tail,
    accumulate, tf32"""
    kv = dict(p.split("=") for p in line.split(":", 1)[1].split())
    K, splitk, path = int(kv["K"]), int(kv["splitk"]), kv["path"]
    chunk = int(kv["kb_per_split" if path == "tc" else "k_chunk"])
    n = (K + 31) // 32 if path == "tc" else K
    return (path, kv["a"], kv["b"], kv["a_row0"] != "0" or kv["b_row0"] != "0", splitk > 1,
            splitk > 1 and n - (splitk - 1) * chunk < chunk, K % 32 != 0, kv["accumulate"] == "1", kv["tf32"] == "1")


_CHILD = r"""
import sys
sys.path[:0] = [{root!r}, {pkg!r}, {tests!r}]
import torch
import b200rnn
from b200rnn.functional import rnn_forward
import test_gpu_grad_gemm_f64 as m
from test_gpu_numerics_f64 import _abi_ln_fused
DEV = "cuda:0"
torch.backends.cuda.matmul.fp32_precision = "ieee"


def mark(what):
    torch.cuda.synchronize()
    print("[b200rnn] phase", what, file=sys.stderr, flush=True)


def backward(kind, I, H, B, T, bi, hx=False, ragged=False, tf32=False, sink=False, frozen=False):
    torch.manual_seed(0)
    cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    mine = b200rnn.from_torch(cls(I, H, bidirectional=bi, batch_first=True)).to(DEV)
    D = 2 if bi else 1
    x = torch.randn(B, T, I, device=DEV, requires_grad=True)
    if frozen:
        mine.weight_ih_l0.requires_grad_(False)
    if sink:   # every gradient view 4 bytes off 16-byte alignment: the weight gradients go to FFMA and accumulate
        ps = [p for p in mine.parameters()]
        flat = torch.zeros(sum(p.numel() + 64 for p in ps), device=DEV)
        views, off = {{}}, 1
        for p in ps:
            views[p.data_ptr()] = flat[off:off + p.numel()].view_as(p)
            off += p.numel() + 64
        mine._grad_sink = lambda weights: [views[w.data_ptr()] for w in weights]
    if hx or ragged or tf32:
        cfg = mine._config()
        cfg.tf32 = tf32
        lens = torch.randint(1, T + 1, (B,)) if ragged else None
        h0 = torch.randn(D, B, H, device=DEV, requires_grad=True) if hx else None
        if hx and kind == "lstm":
            h0 = (h0, torch.randn(D, B, H, device=DEV, requires_grad=True))
        out = rnn_forward(x, mine._flat_weights, cfg, lengths=lens, hx=h0)   # cfg.batch_first, as the module
        out[0].sum().backward()
    else:
        mine(x)[0].sum().backward()


mark("backward")
for fam, (I, H, B, T, G) in m.FAMILIES.items():
    kind = "gru" if G == 3 else "lstm"
    for bi in (False, True):
        backward(kind, I, H, B, T, bi)
        backward(kind, I, H, B, T, bi, hx=True)
        backward(kind, I, H, B, T, bi, tf32=True)
        backward(kind, I, H, B, T, bi, sink=True)
    backward(kind, I, H, B, T, False, ragged=True)
    backward(kind, I, H, B, T, True, frozen=True)
    if kind == "gru":   # the LayerNorm prologue of the model shell (C ABI, saved LN(x) as the dW_ih operand)
        gru = b200rnn.GRU(I, H).to(DEV)
        lens = torch.randint(1, T + 1, (B,))
        ln_w, ln_b = torch.ones(I, device=DEV), torch.zeros(I, device=DEV)
        _abi_ln_fused(torch.randn(T, B, I, device=DEV), lens, gru, ln_w, ln_b, torch.randn(T, B, H, device=DEV))
mark("matrix")
for table in (m.GENERIC, m.REAL):
    for name, (prog, tf32) in table.items():
        m._program(prog, tf32, check=False)
mark("end")
"""


def test_matrix_covers_every_mode_of_the_backward():
    env = dict(os.environ, B200RNN_DEBUG="1")
    code = _CHILD.format(root=ROOT, pkg=PKG, tests=os.path.join(ROOT, "tests"))
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout + proc.stderr[-4000:]
    phase, seen = None, {"backward": set(), "matrix": set()}
    for ln in proc.stderr.splitlines():
        if ln.startswith("[b200rnn] phase "):
            phase = ln.split()[-1]
        elif ln.startswith("[b200rnn] grad gemm ") and phase in seen:
            seen[phase].add(_tuple(ln))
    print("backward modes (path, a, b, row0 != 0, split-K, short last split, K tail, accumulate, tf32):")
    for t in sorted(seen["backward"]):
        print("  ", t)
    assert seen["backward"], proc.stderr[-4000:]
    missing = seen["backward"] - seen["matrix"]
    assert not missing, sorted(missing)
