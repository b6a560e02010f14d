"""The split classification head of ``FusedFuseStep``: the audio half of the head runs on the audio stream before the
join, each branch emits its halves of the row logits, and after the join one single-CTA launch does the loss, dW and
Adam. It must compute exactly what the one-launch head computes: same logits, loss, ``fc_final.0.weight`` and Adam
state, bit for bit, in train mode with dropout, eager and under CUDA-graph replay.
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T_A, E_A, H_A, T_T, E_T, H_T = 120, 256, 256, 30, 1024, 128


def _model(p, regression=False):
    import b200rnn

    torch.manual_seed(0)
    m = b200rnn.fusion_net(text_embed_size=E_T, text_hidden_dims=H_T, rnn_layers=2, dropout=p,
                           num_classes=1 if regression else 2, audio_hidden_dims=H_A, audio_embed_size=E_A,
                           regression=regression).to(DEV)
    for q in m.parameters():
        q.requires_grad = False
    m.fc_final[0].weight.requires_grad = True
    m.train()
    return m


def _batches(B, n, seed=99):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(B, T_A, E_A, generator=g).to(DEV), torch.randn(B, T_T, E_T, generator=g).to(DEV),
             torch.randint(0, 2, (B,), generator=g).to(DEV)) for _ in range(n)]


def _state(step, out, loss):
    return [out.clone(), loss.clone(), step.w.detach().clone(), step.m.clone(), step.v.clone(),
            step.step_count.clone(), step.rng_state.clone()]


def _assert_bitwise(a, b, what):
    names = ["logits", "loss", "fc_final.0.weight", "adam m", "adam v", "adam step", "rng state"]
    for n, x, y in zip(names, a, b):
        assert torch.equal(x, y), f"{what}: {n} differs (max abs {(x.double() - y.double()).abs().max().item()})"


@pytest.mark.parametrize("B", [128, 96])
def test_split_head_equals_one_launch_head_bitwise(B):
    import b200rnn

    m0 = _model(0.3)
    m1 = copy.deepcopy(m0)
    split = b200rnn.FusedFuseStep(m0, lr=1e-3, exchange="none")
    whole = b200rnn.FusedFuseStep(m1, lr=1e-3, exchange="none")
    assert split.split_loss
    whole.split_loss = False           # the one-launch head after the join
    for i, (a, t, y) in enumerate(_batches(B, 4)):
        o0, l0 = split(b200rnn.FuseBatch(a, t), y)
        o1, l1 = whole(b200rnn.FuseBatch(a, t), y)
        torch.cuda.synchronize()
        assert torch.isfinite(l0).item()
        _assert_bitwise(_state(split, o0, l0), _state(whole, o1, l1), f"B={B} step {i}")
    assert not torch.equal(m0.fc_final[0].weight, _model(0.3).fc_final[0].weight)   # the update did run


def test_split_head_graph_replay_equals_eager():
    import b200rnn

    m0 = _model(0.3)
    m1 = copy.deepcopy(m0)
    eager = b200rnn.FusedFuseStep(m0, lr=1e-3, exchange="none")
    graphed = b200rnn.FusedFuseStep(m1, lr=1e-3, exchange="none")
    (a, t, y), = _batches(128, 1, seed=7)
    batch = b200rnn.FuseBatch(a, t)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):      # one eager warm-up step on each (lazy streams, scratch, kernel attributes)
        graphed(batch, y)
    torch.cuda.current_stream().wait_stream(side)
    eager(batch, y)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        go, gl = graphed(batch, y)
    for i in range(3):
        g.replay()
        eo, el = eager(batch, y)
        torch.cuda.synchronize()
        _assert_bitwise(_state(graphed, go, gl), _state(eager, eo, el), f"replay {i}")


def test_split_head_only_for_classification():
    import b200rnn

    assert not b200rnn.FusedFuseStep(_model(0.3, regression=True), exchange="none").split_loss
    assert not b200rnn.FusedFuseStep(_model(0.3), exchange="none", concurrent_branches=False).split_loss
