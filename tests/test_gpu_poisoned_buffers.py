"""Every recurrence entry on dirty buffers: nothing the library computes may depend on what the allocator hands it.

The reserve, the scratch, y, h_n / c_n, dx, dh_0 / dc_0 and the weight-gradient buffer all come from torch.empty /
torch.empty_like in b200rnn/functional.py. Several results hold only if a kernel writes something before anything reads
it: the zeroed gate gradients of the steps a ragged cluster skips, the per-slice bias partials, dh_0 of a cluster that
ran no step, the streamed input projection's ready counters. Lose one of those writes and the suite still passes
whenever the allocator returns zeros or stale finite data. Here functional.py's `torch` is wrapped so that empty /
empty_like return buffers filled with one 32-bit word, and each case runs forward and backward twice: once with the word
0x7FC00000 and once with 0. Every output and gradient must be bitwise equal between the two runs, and finite.

0x7FC00000 is a NaN as a float (and its 16-bit halves are 0 and a NaN in fp16 and bf16), so an unwritten float that is
read reaches the result. As an int it is a large positive number: a ready counter that is not reset lets the recurrence's
`ready < tiles_n` wait pass before the GEMM has written the tile, and the numbers change instead of the kernel spinning
(0xFF bytes would read -1 and spin). Two buffers are read as ints and made safe by the library: the ragged batch's slot
order (launch_length_order writes it first in the forward and in the backward) and the ready counters (zeroed before any
streamed GEMM, by the kernel that writes the GEMM's A operand or by a memset).

Cases: every fixed plan_rec_fwd / plan_rec_bwd entry (test_gpu_numerics_f64.CONFIGS), every runtime-sized instantiation
of test_gpu_anyh_numerics_f64.CONFIGS in fp32, fp16 and bf16, ragged and fixed-length, with hx and dh_0 / dc_0, and two
layers with and without inter-layer dropout (the dropout generator's state is restored before each run, so both draw the
same mask)."""
import pytest
import torch

from test_gpu_anyh_numerics_f64 import CONFIGS as ANYH_CONFIGS
from test_gpu_numerics_f64 import CONFIGS as FIXED_CONFIGS
from test_gpu_numerics_f64 import _ragged_lengths

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
POISON = 0x7FC00000


class _FilledTorch:
    """`torch` for b200rnn.functional: empty / empty_like return buffers whose every 32-bit word is `word`"""

    def __init__(self, word):
        self._word = word

    def __getattr__(self, name):
        return getattr(torch, name)

    def _fill(self, t):
        s = t.untyped_storage()
        n = s.nbytes()
        if n:
            b = torch.empty(0, dtype=torch.uint8, device=t.device).set_(s)
            n4 = n // 4 * 4
            b[:n4].view(torch.int32).fill_(self._word)
            tail = torch.tensor(list(self._word.to_bytes(4, "little")), dtype=torch.uint8)[:n - n4]
            b[n4:].copy_(tail)
        return t

    def empty(self, *args, **kwargs):
        return self._fill(torch.empty(*args, **kwargs))

    def empty_like(self, *args, **kwargs):
        return self._fill(torch.empty_like(*args, **kwargs))


def _stock(kind, I, H, L, bi, P=0, dropout=0.0):
    if kind in ("gru", "lstm"):
        cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
        return cls(I, H, num_layers=L, bidirectional=bi, dropout=dropout, **({"proj_size": P} if P else {}))
    return torch.nn.RNN(I, H, num_layers=L, nonlinearity=kind[4:], bidirectional=bi, dropout=dropout)


def _case(kind, I, H, B, bi, *, P=0, L=1, dtype=torch.float32, ragged=False, hx=True, tf32=False, fused=False,
          dropout=0.0, T=12):
    """one forward + backward per fill word: {name: tensor} of every output and gradient of each run"""
    import b200rnn
    from b200rnn import functional
    from b200rnn.functional import rnn_forward, rnn_forward_fused

    torch.manual_seed(0)
    ref = _stock(kind, I, H, L, bi, P, dropout)
    D, HO = (2 if bi else 1), (P or H)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(T, B, I, generator=g)
    lens = _ragged_lengths(B, T) if ragged else None
    states = [0.5 * torch.randn(L * D, B, HO, generator=g)] + (
        [0.5 * torch.randn(L * D, B, H, generator=g)] if kind == "lstm" else [])
    wy = torch.randn(T, B, D * HO, generator=g)
    ws = [torch.randn(s.shape, generator=g) for s in states]
    mine = b200rnn.from_torch(ref).to(DEV, dtype).train(dropout > 0)
    rng0 = mine._rng_state.clone()
    results = []
    for word in (POISON, 0):
        saved = functional.torch
        functional.torch = _FilledTorch(word)
        try:
            mine.zero_grad(set_to_none=True)
            mine._rng_state.copy_(rng0)
            cfg = mine._config()
            cfg.tf32 = tf32
            xm = x.to(DEV, dtype).requires_grad_(not fused)
            if fused:   # the no-grad fused forward: no initial state, fixed length
                out = rnn_forward_fused(xm, mine._flat_weights, cfg)
                res = dict(zip(("y", "h_n", "c_n"), out))
            else:
                st = [s.to(DEV, dtype).requires_grad_(True) for s in states] if hx else []
                h = None if not hx else (tuple(st) if kind == "lstm" else st[0])
                out = rnn_forward(xm, mine._flat_weights, cfg, mine._rng_state, lengths=lens, hx=h)
                loss = (out[0] * wy.to(DEV, dtype)).sum() + sum((s * w.to(DEV, dtype)).sum()
                                                               for s, w in zip(out[1:], ws))
                loss.backward()
                res = dict(zip(("y", "h_n", "c_n"), out))
                res["dx"] = xm.grad
                res.update({"d" + n: p.grad for n, p in mine.named_parameters()})
                res.update(dict(zip(("dh_0", "dc_0"), (s.grad for s in st))))
            torch.cuda.synchronize()
            results.append({k: v.detach().clone() for k, v in res.items()})
        finally:
            functional.torch = saved
    return results


def _check(results, what):
    dirty, clean = results
    assert sorted(dirty) == sorted(clean)
    for k, v in clean.items():
        assert torch.isfinite(dirty[k]).all(), (what, k, "not finite on poisoned buffers")
        assert torch.equal(dirty[k], v), (what, k, "differs between poisoned and zeroed buffers")


def test_fill_word_reaches_every_byte():
    """the proxy itself: fp32 / int32 words, and the 16-bit halves of a buffer whose size is not a multiple of 4"""
    ft = _FilledTorch(POISON)
    a = ft.empty(7, device=DEV)
    assert torch.isnan(a).all() and (a.view(torch.int32) == POISON).all()
    h = ft.empty(5, dtype=torch.float16, device=DEV)
    assert h.view(torch.int16).cpu().tolist() == [0, 0x7FC0, 0, 0x7FC0, 0]
    e = ft.empty_like(torch.zeros(3, 4, device=DEV).t())
    assert (e.contiguous().view(torch.int32) == POISON).all()


@pytest.mark.parametrize("ragged", [False, True], ids=["fixed", "ragged"])
@pytest.mark.parametrize("name", list(FIXED_CONFIGS))
def test_fixed_configs(name, ragged):
    kind, I, H, B, bi, P, mode = FIXED_CONFIGS[name]
    fused = mode == "f16"
    if fused and ragged:
        pytest.skip("the fp16-pair forward is the no-grad fused entry, fixed-length")
    _check(_case(kind, I, H, B, bi, P=P, ragged=ragged, hx=not fused, tf32=mode == "tf32", fused=fused),
           (name, ragged))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("ragged", [False, True], ids=["fixed", "ragged"])
@pytest.mark.parametrize("name", list(ANYH_CONFIGS))
def test_runtime_sized(name, ragged, dtype):
    kind, I, H, B, bi, _ = ANYH_CONFIGS[name]
    _check(_case(kind, I, H, B, bi, dtype=dtype, ragged=ragged), (name, ragged, dtype))


@pytest.mark.parametrize("dropout", [0.0, 0.3], ids=["nodrop", "dropout"])
@pytest.mark.parametrize("kind, I, H, B, bi, ragged", [
    ("gru", 256, 256, 64, False, False),    # the fixed GRU-256 config with the streamed input projection
    ("gru", 256, 256, 64, False, True),
    ("lstm", 64, 464, 12, True, True),      # runtime-sized, L2 tier
    ("rnn_tanh", 40, 272, 16, True, True),
], ids=["gru256", "gru256_ragged", "lstm464_bi_ragged", "tanh272_bi_ragged"])
def test_two_layers(kind, I, H, B, bi, ragged, dropout):
    _check(_case(kind, I, H, B, bi, L=2, ragged=ragged, dropout=dropout), (kind, H, ragged, dropout))

