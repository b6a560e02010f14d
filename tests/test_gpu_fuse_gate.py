"""The fuse step gates its text stream on the audio prologue: ``b200rnn_forward_fused`` records the caller's
``prologue_done`` event once the layer-0 operand preparation is enqueued, before the first GEMM, and the text branch
waits on it (b200rnn/fused_head.py ``_encoders``). The event must be recorded early (else the text branch would wait
for the whole audio chain), and the gated two-stream step must capture into a CUDA graph that replays bit for bit
what an eager call computes."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_prologue_event_is_recorded_before_the_first_gemm():
    import b200rnn
    from b200rnn.functional import rnn_forward_fused

    torch.manual_seed(0)
    gru = b200rnn.GRU(256, 256, num_layers=2, batch_first=True).to(DEV)
    ln = torch.nn.LayerNorm(256).to(DEV)
    x = torch.randn(128, 120, 256, device=DEV)
    ref = rnn_forward_fused(x, gru._flat_weights, gru._config(), None, ln.weight, ln.bias, ln.eps, pool_sum=True)[0]
    begin, prologue, end = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    prologue.record()       # an earlier record: if the call did not record it again, it would precede `begin`
    torch.cuda._sleep(20_000_000)   # ~10 ms: the whole call is enqueued before the device reaches `begin`
    begin.record()
    out = rnn_forward_fused(x, gru._flat_weights, gru._config(), None, ln.weight, ln.bias, ln.eps, pool_sum=True,
                            prologue_done=prologue)[0]
    end.record()
    torch.cuda.synchronize()
    assert 0 < begin.elapsed_time(prologue) < 0.25 * begin.elapsed_time(end)
    assert torch.equal(out, ref)


@pytest.mark.parametrize("regression", [False, True])
def test_two_stream_features_replay_bitwise_equal_to_eager(regression):
    import b200rnn

    torch.manual_seed(1)
    m = b200rnn.fusion_net(1024, 128, 2, 0.3, 1 if regression else 2, 256, 256, regression=regression).to(DEV)
    for p in m.parameters():
        p.requires_grad = False
    m.fc_final[0].weight.requires_grad = True
    m.eval()
    step = b200rnn.FusedFuseStep(m, exchange="none", concurrent_branches=True)
    B = 128
    audio = torch.randn(B, 120, 256, device=DEV)
    text = torch.randn(B, 30, 1024, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step.features(b200rnn.FuseBatch(audio, text))
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_tf, static_af = step.features(b200rnn.FuseBatch(audio, text))
    for i in range(50):
        a, t = torch.randn_like(audio), torch.randn_like(text)
        audio.copy_(a)
        text.copy_(t)
        graph.replay()
        tf, af = step.features(b200rnn.FuseBatch(a, t))
        torch.cuda.synchronize()
        assert torch.equal(static_tf, tf) and torch.equal(static_af, af), f"replay {i} differs from the eager call"
