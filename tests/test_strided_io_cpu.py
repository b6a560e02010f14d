"""The fused LayerNorm's operand check (functional._ln_operand_ok): the prologue and its backward read x in place with
float4 loads, so the Python entries pass it a dense copy of any x whose base or row strides are not 16-byte multiples,
and of a gamma / beta that is not 16-byte aligned. CPU tensors: the check is pointer and stride arithmetic only."""
import pytest
import torch

from b200rnn import functional as F

T, B, I = 3, 4, 8


def _view(st, sb, off=0, n=None):
    buf = torch.zeros(n or (off + T * abs(st) + B * abs(sb) + I + 64))
    assert buf.data_ptr() % 16 == 0
    return buf.as_strided((T, B, I), (st, sb, 1), off)


@pytest.mark.parametrize("st,sb,off", [
    (B * I, I, 0),              # dense time-major
    (I, T * I, 0),              # batch-first, transposed to time-major
    (B * (I + 8), I + 8, 0),    # feature slice of a wider row, aligned
    (2 * B * I, 2 * I, 0),      # batch gap
    (2 * B * I, I, 0),          # time gap
    (I, 0, 0),                  # one sequence broadcast over the batch
    (0, I, 0),                  # one step broadcast over time
    (B * I, I, 4),              # offset by a whole float4
])
def test_aligned_views_are_read_in_place(st, sb, off):
    x = _view(st, sb, off)
    g = torch.ones(I)
    assert F._ln_operand_ok(x, g, torch.zeros(I))
    assert F._ln_operand_ok(x, None, None)
    x2, g2, b2 = F._ln_operands(x, g, None)
    assert x2 is x and g2 is g and b2 is None


@pytest.mark.parametrize("st,sb,off", [
    (B * (I + 8), I + 8, 1),    # feature slice at offset 1: misaligned base
    (B * (I + 8), I + 8, 2),
    (B * (I + 1), I + 1, 0),    # row stride not a multiple of 4
    (3, I, 0),                  # time stride 3
    (B * I + 2, I, 0),          # time stride off by 2
    (B * I, I + 2, 0),          # batch stride off by 2
])
def test_unaligned_views_get_a_dense_copy(st, sb, off):
    x = _view(st, sb, off).copy_(torch.randn(T, B, I))
    g, b = torch.randn(I), torch.randn(I)
    assert not F._ln_operand_ok(x, g, b)
    x2, g2, b2 = F._ln_operands(x, g, b)
    assert x2.is_contiguous() and x2.data_ptr() % 16 == 0 and x2.data_ptr() != x.data_ptr()
    assert torch.equal(x2, x)
    assert g2 is g and b2 is b
    assert F._ln_operand_ok(x2, g2, b2)


def test_size_one_dims_follow_the_strides_the_library_checks():
    """T = 1 with a time stride of 3 and B = 1 with a batch stride of 1: the C side checks both strides whatever the
    extent, so these take the copy too (never an UNSUPPORTED from the library)"""
    buf = torch.zeros(256)
    assert not F._ln_operand_ok(buf.as_strided((1, B, I), (3, I, 1)), None, None)
    assert not F._ln_operand_ok(buf.as_strided((T, 1, I), (I, 1, 1)), None, None)
    assert F._ln_operand_ok(buf.as_strided((T, 1, I), (I, 4, 1)), None, None)


@pytest.mark.parametrize("which", ["gamma", "beta"])
def test_unaligned_affine_parameters_are_copied(which):
    x = _view(B * I, I)
    p = torch.randn(I + 1)[1:]
    assert p.data_ptr() % 16 != 0
    g, b = (p, torch.ones(I)) if which == "gamma" else (torch.ones(I), p)
    assert not F._ln_operand_ok(x, g, b)
    x2, g2, b2 = F._ln_operands(x, g, b)
    assert F._ln_operand_ok(x2, g2, b2)
    assert torch.equal(g2, g) and torch.equal(b2, b)
    assert x2 is x   # x itself is readable in place: only the parameter is copied
    assert (g2 is g) == (which == "beta") and (b2 is b) == (which == "gamma")


def test_copies_carry_gradients_back_to_the_callers_tensors():
    base = torch.randn(T * B * (I + 8) + 1, requires_grad=True)
    x = base.as_strided((T, B, I), (B * (I + 8), I + 8, 1), 1)
    g = torch.randn(I + 1, requires_grad=True)
    gv = g[1:]
    x2, g2, _ = F._ln_operands(x, gv, None)
    (x2 * torch.arange(T * B * I, dtype=torch.float32).view(T, B, I)).sum().backward(retain_graph=True)
    want = torch.zeros(T * B * (I + 8) + 1)
    want.as_strided((T, B, I), (B * (I + 8), I + 8, 1), 1).copy_(torch.arange(T * B * I, dtype=torch.float32).view(T, B, I))
    assert torch.equal(base.grad, want)
    (g2 * 2).sum().backward()
    assert torch.equal(g.grad, torch.tensor([0.0] + [2.0] * I))
