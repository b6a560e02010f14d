"""Single-pass TF32 mode without a GPU: how the mode follows torch's fp32 matmul precision, the descriptor flag, the
float64 emulation oracle (oracle/tf32.py) and the SASS of the TF32 kernel instantiations."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from b200rnn import _lib
from b200rnn.functional import RNNConfig, _make_desc, tf32_enabled

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _knobs():
    b = torch.backends
    return [(b, "fp32_precision"), (b.cuda.matmul, "fp32_precision"), (b.cudnn, "fp32_precision"),
            (b.cudnn.conv, "fp32_precision"), (b.cudnn.rnn, "fp32_precision"), (b.mkldnn, "fp32_precision"),
            (b.mkldnn.matmul, "fp32_precision"), (b.mkldnn.conv, "fp32_precision"), (b.mkldnn.rnn, "fp32_precision")]


@pytest.fixture
def precision():
    """Saves torch's fp32 precision settings and restores them after the test (the global one first: setting it
    propagates to the backends)."""
    saved = [(obj, name, getattr(obj, name)) for obj, name in _knobs()]
    yield torch.backends
    for obj, name, value in saved:
        setattr(obj, name, value)


def test_default_is_off(precision):
    precision.fp32_precision = "none"
    precision.cuda.matmul.fp32_precision = "none"
    assert not tf32_enabled()


def test_legacy_api(precision):
    torch.set_float32_matmul_precision("high")
    assert tf32_enabled()
    torch.set_float32_matmul_precision("highest")
    assert not tf32_enabled()


def test_new_api(precision):
    precision.cuda.matmul.fp32_precision = "tf32"
    assert tf32_enabled()
    precision.cuda.matmul.fp32_precision = "ieee"
    assert not tf32_enabled()
    # mixing both APIs in one process: torch.get_float32_matmul_precision() would raise here, tf32_enabled() does not
    torch.set_float32_matmul_precision("high")
    assert tf32_enabled()


def test_none_falls_back_to_the_global_setting(precision):
    precision.fp32_precision = "tf32"
    precision.cuda.matmul.fp32_precision = "none"
    assert tf32_enabled()
    precision.fp32_precision = "ieee"
    precision.cuda.matmul.fp32_precision = "none"
    assert not tf32_enabled()


def test_cudnn_rnn_setting_is_not_followed(precision):
    precision.fp32_precision = "none"
    precision.cuda.matmul.fp32_precision = "none"
    precision.cudnn.rnn.fp32_precision = "tf32"
    assert not tf32_enabled()


def test_module_config_follows_the_setting(precision):
    import b200rnn

    m = b200rnn.GRU(256, 256, num_layers=2)
    precision.cuda.matmul.fp32_precision = "ieee"
    assert not m._config().tf32
    precision.cuda.matmul.fp32_precision = "tf32"
    assert m._config().tf32


def _cfg(tf32):
    return RNNConfig(mode=_lib.GRU, input_size=256, hidden_size=256, num_layers=2, num_dirs=1, dropout=0.0,
                     training=False, batch_first=True, tf32=tf32)


def test_desc_flag():
    for save in (False, True):
        for acc in (False, True):
            for ln in (False, True):
                off = _make_desc(_cfg(False), 4, 5, save, acc, ln).flags
                on = _make_desc(_cfg(True), 4, 5, save, acc, ln).flags
                assert off & _lib.FLAG_TF32 == 0
                assert on == off | _lib.FLAG_TF32
    assert _lib.FLAG_TF32 == 8


def test_header_flag_matches_binding():
    with open(os.path.join(ROOT, "include", "b200rnn.h")) as f:
        m = re.search(r"#define\s+B200RNN_FLAG_TF32\s+(\d+)u", f.read())
    assert m and int(m.group(1)) == _lib.FLAG_TF32


# ---- the emulation oracle ----------------------------------------------------------------------------------------

def test_round_tf32_hand_picked_values():
    from oracle.tf32 import round_tf32

    ulp = 2.0 ** -10                       # TF32 spacing in [1, 2)
    cases = [
        (1.0, 1.0),                        # already TF32
        (1.0 + ulp, 1.0 + ulp),
        (-(1.0 + 3 * ulp), -(1.0 + 3 * ulp)),
        (1.0 + ulp / 2, 1.0 + ulp),        # tie: away from zero
        (-(1.0 + ulp / 2), -(1.0 + ulp)),
        (1.0 + 3 * ulp / 2, 1.0 + 2 * ulp),  # tie above an odd mantissa: away from zero too (not to even)
        (1.0 + ulp / 2 - 2.0 ** -23, 1.0),  # just below the tie
        (1.0 + ulp / 2 + 2.0 ** -23, 1.0 + ulp),
        (-(1.0 + ulp / 2 - 2.0 ** -23), -1.0),
        (2.0 - ulp / 2, 2.0),              # rounds up into the next binade
        (0.0, 0.0),
        (3.0 * 2.0 ** -130, 3.0 * 2.0 ** -130),  # subnormal with few bits
    ]
    x = np.array([c[0] for c in cases], dtype=np.float32)
    want = np.array([c[1] for c in cases], dtype=np.float32)
    got = round_tf32(x)
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, want)
    assert np.signbit(round_tf32(np.float32(-0.0)))
    # idempotent, and the 13 low bits are clear
    r = round_tf32(np.random.default_rng(0).standard_normal(1000).astype(np.float32))
    np.testing.assert_array_equal(round_tf32(r), r)
    assert not (r.view(np.uint32) & 0x1FFF).any()


@pytest.mark.parametrize("kind, bi, lengths", [("gru", False, None), ("lstm", True, None), ("gru", True, [5, 3, 1]),
                                                ("lstm", False, [2, 5, 4])])
def test_emulation_without_rounding_is_rnn_numpy(kind, bi, lengths):
    from oracle.rnn_numpy import NumpyRNN
    from oracle.tf32 import Tf32RNN

    torch.manual_seed(0)
    cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    ref = cls(12, 8, num_layers=2, bidirectional=bi)
    w = [p.detach().double().numpy() for p in ref.parameters()]
    rng = np.random.default_rng(1)
    x = rng.standard_normal((5, 3, 12))
    a, b = NumpyRNN(kind, w, 2, bi), Tf32RNN(kind, w, 2, bi, rec_round=True, rounding=False)
    outs_a, outs_b = a.forward(x, lengths), b.forward(x, lengths)
    for u, v in zip(outs_a, outs_b):
        np.testing.assert_array_equal(u, v)
    dy = rng.standard_normal(outs_a[0].shape)
    dh = rng.standard_normal(outs_a[1].shape)
    dxa, ga = a.backward(dy, dh)
    dxb, gb = b.backward(dy, dh)
    np.testing.assert_array_equal(dxa, dxb)
    for u, v in zip(ga, gb):
        np.testing.assert_array_equal(u, v)


def test_emulation_with_rounding_is_close_to_but_not_fp64():
    from oracle.rnn_numpy import NumpyRNN
    from oracle.tf32 import Tf32RNN

    torch.manual_seed(0)
    ref = torch.nn.GRU(64, 32, num_layers=1)
    w = [p.detach().double().numpy() for p in ref.parameters()]
    x = np.random.default_rng(2).standard_normal((6, 4, 64))
    y64 = NumpyRNN("gru", w, 1, False).forward(x)[0]
    y_gemm = Tf32RNN("gru", w, 1, False, rec_round=False).forward(x)[0]
    y_all = Tf32RNN("gru", w, 1, False, rec_round=True).forward(x)[0]
    e_gemm, e_all = np.abs(y_gemm - y64).max(), np.abs(y_all - y64).max()
    assert 1e-6 < e_gemm < 1e-2 and 1e-6 < e_all < 1e-2
    assert not np.array_equal(y_gemm, y_all)


# ---- SASS of the TF32 instantiations -------------------------------------------------------------------------------

cuobjdump = shutil.which("cuobjdump") or shutil.which("/usr/local/cuda/bin/cuobjdump")


@pytest.fixture(scope="module")
def sass():
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    out, name = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name is not None:
            m = re.search(r"\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                out[name].append(m.group(1))
    return out


def _count(ops, prefix):
    return sum(1 for o in ops if o.startswith(prefix))


def test_tc8_tf32_issues_a_third_of_the_hmma(sass):
    x3 = {k: v for k, v in sass.items() if "rec_fwd_tc_kernel" in k}
    t1 = {k: v for k, v in sass.items() if "rec_fwd_tf32_kernel" in k}
    assert len(x3) == 2 and len(t1) == 2, (sorted(x3), sorted(t1))
    for vl in ("ILb0E", "ILb1E"):
        (a,) = [v for k, v in x3.items() if vl in k]
        (b,) = [v for k, v in t1.items() if vl in k]
        n3, n1 = _count(a, "HMMA.1688.F32.TF32"), _count(b, "HMMA.1688.F32.TF32")
        assert n1 > 0 and 3 * n1 == n3, (vl, n3, n1)


def test_gemm_tf32_issues_a_third_of_the_wgmma(sass):
    gemm = {re.search(r"gemm_tf32x3_kernelILb(\d)ELb(\d)E", k).groups(): v for k, v in sass.items()
            if "gemm_tf32x3_kernel" in k}
    assert set(gemm) == {("0", "0"), ("0", "1"), ("1", "0"), ("1", "1")}, sorted(gemm)
    for mn in ("0", "1"):
        n3, n1 = _count(gemm[(mn, "0")], "HGMMA"), _count(gemm[(mn, "1")], "HGMMA")
        assert n1 > 0 and 3 * n1 == n3, (mn, n3, n1)


def test_tf32_instantiations_keep_everything_in_registers(sass):
    new = {k: v for k, v in sass.items()
           if "rec_fwd_tf32_kernel" in k or re.search(r"gemm_tf32x3_kernelILb\dELb1E", k)}
    assert len(new) == 4, sorted(new)
    for name, ops in new.items():
        local = sorted({o for o in ops if o.startswith(("LDL", "STL"))})
        assert not local, f"{name}: local-memory traffic {local}"
