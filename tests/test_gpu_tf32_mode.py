"""Single-pass TF32 mode on the GPU (torch's fp32 matmul precision "tf32" -> B200RNN_FLAG_TF32).

Oracle: oracle/tf32.py, a float64 GRU / LSTM that rounds exactly the operands the kernels round (input projection,
weight- and input-gradient GEMMs, and W_hh h_{t-1} in the GRU-256 tensor-core recurrence tc8), teacher-forced with the
per-layer outputs the kernels produced so that it rounds the same fp32 values they rounded. Against it the GPU result
must meet the fp32-level bounds the default 3xTF32 path meets against oracle/rnn_numpy.py (outputs 1e-5 abs, gradients
1e-4 relative to the largest entry): the kernels do single-pass TF32 and nothing looser. The error against exact fp64
is printed, not asserted.

Which recurrence config runs depends on the batch (csrc/rnn_rec.cu plan_rec_fwd, 30 co-resident 4-CTA clusters on a
132-SM H100): B = 128 takes tc8 with the input projection streamed into it, B = 160 tc8 after it, B <= 64 an FFMA
config (bs4 / bs2), whose recurrence stays fp32 - there only the GEMMs change.
"""
import contextlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OUT_TOL = 1e-5
GRAD_RTOL = 1e-4
FEAT_TOL = 1e-4     # sums over time / logits, as in tests/test_gpu_fuse_parity.py


@contextlib.contextmanager
def matmul_precision(mode):
    """torch.backends.cuda.matmul.fp32_precision = mode inside the block (the global setting stays "none")."""
    b = torch.backends
    saved = (b.fp32_precision, b.cuda.matmul.fp32_precision)
    b.cuda.matmul.fp32_precision = mode
    try:
        yield
    finally:
        b.fp32_precision = saved[0]
        b.cuda.matmul.fp32_precision = saved[1]


def _relmax(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _absmax(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _np(t):
    return t.detach().cpu().double().numpy()


def _one_layer(kind, params, I, H, bi):
    import b200rnn

    m = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(I, H, num_layers=1, bidirectional=bi).to(DEV).eval()
    with torch.no_grad():
        for q, src in zip(m._flat_weights, params):
            q.copy_(src)
    return m


def _layer_outputs(kind, ref, L, bi, x, lengths, y_last):
    """What the kernels output per layer in TF32 mode, time-major: layers 0..L-2 from one-layer modules with the same
    weights (the kernels of the L-layer call, on the same input), the last one the L-layer call's own output."""
    from b200rnn.functional import rnn_forward

    D = 2 if bi else 1
    params = list(ref.parameters())
    outs, inp = [], x
    for l in range(L - 1):
        m = _one_layer(kind, params[4 * D * l:4 * D * (l + 1)], inp.shape[-1], ref.hidden_size, bi)
        with torch.no_grad(), matmul_precision("tf32"):
            inp = rnn_forward(inp, m._flat_weights, m._config(), lengths=lengths)[0]
        outs.append(_np(inp))
    outs.append(_np(y_last))
    return outs


CASES = [
    # id, kind, B, T, I, H, L, bi, tc8, ragged
    ("gru256_b128_tc8_streamed", "gru", 128, 120, 256, 256, 2, False, True, False),
    ("gru256_b160_tc8_serial", "gru", 160, 40, 256, 256, 2, False, True, False),
    ("gru256_b64_bs4", "gru", 64, 60, 256, 256, 2, False, False, False),
    ("bilstm128_text", "lstm", 48, 30, 1024, 128, 2, True, False, False),
    ("bilstm256_text", "lstm", 32, 30, 1024, 256, 2, True, False, False),
    ("gru256_b128_tc8_ragged", "gru", 128, 60, 256, 256, 2, False, True, True),
    ("bilstm128_ragged", "lstm", 24, 20, 1024, 128, 2, True, False, True),
]


@pytest.mark.parametrize("kind, B, T, I, H, L, bi, tc8, ragged", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_tf32_mode_matches_emulation(kind, B, T, I, H, L, bi, tc8, ragged):
    import b200rnn
    from b200rnn.functional import rnn_forward
    from oracle.rnn_numpy import NumpyRNN
    from oracle.tf32 import Tf32RNN

    torch.manual_seed(0)
    ref = (torch.nn.GRU if kind == "gru" else torch.nn.LSTM)(I, H, num_layers=L, bidirectional=bi)
    mine = b200rnn.from_torch(ref).to(DEV).eval()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(T, B, I, generator=g)
    lengths = None
    if ragged:
        lengths = torch.randint(1, T + 1, (B,), generator=g)
        lengths[B // 3] = T
    xm = x.to(DEV).requires_grad_(True)
    with matmul_precision("tf32"):
        cfg = mine._config()
        assert cfg.tf32
        out = rnn_forward(xm, mine._flat_weights, cfg, lengths=lengths)
    states = out[1:]
    dy = torch.randn(out[0].shape, generator=g)
    dstates = [torch.randn(s.shape, generator=g) for s in states]
    loss = (out[0] * dy.to(DEV)).sum() + sum((s * d.to(DEV)).sum() for s, d in zip(states, dstates))
    loss.backward()        # outside the block: the backward follows its forward's mode
    torch.cuda.synchronize()

    w64 = [p.detach().double().numpy() for p in ref.parameters()]
    lens = None if lengths is None else lengths.numpy()
    observed = _layer_outputs(kind, ref, L, bi, x.to(DEV), lengths, out[0])
    errs, errs64 = {}, {}
    for name, orc, dst in (("emu", Tf32RNN(kind, w64, L, bi, rec_round=tc8), errs),
                           ("fp64", NumpyRNN(kind, w64, L, bi), errs64)):
        res = orc.forward(x.double().numpy(), lens, *([observed] if name == "emu" else []))
        dst["y"] = _absmax(_np(out[0]), res[0])
        for i, (s, r) in enumerate(zip(states, res[1:])):
            dst[f"state{i}"] = _absmax(_np(s), r)
        dx, dps = orc.backward(dy.double().numpy(), *[d.double().numpy() for d in dstates])
        dst["dx"] = _relmax(_np(xm.grad), dx)
        for (n, _), p, d in zip(ref.named_parameters(), mine._flat_weights, dps):
            dst["d" + n] = _relmax(_np(p.grad), d)
    print(f"TF32 {kind} B{B} T{T} H{H}: vs emulation {max(errs.values()):.2e}, vs fp64 "
          f"y {errs64['y']:.2e} grads {max(v for k, v in errs64.items() if k.startswith('d')):.2e}")
    for k, v in errs.items():
        tol = OUT_TOL if (k == "y" or k.startswith("state")) else GRAD_RTOL
        assert v <= tol, f"{k}: {v:.3e} > {tol:.0e} (all: {errs})"
    # and the mode is really on: single-pass TF32 is visibly further from fp64 than 3xTF32 (~1e-6) is
    assert errs64["y"] > 1e-5, errs64


def test_fused_layernorm_time_sum_matches_emulation():
    """The audio branch of the fuse model: LayerNorm folded into the layer-0 projection, sum over time in the last
    recurrence, forward (no grad: b200rnn_forward_fused) and training graph (b200rnn_backward_fused)."""
    import b200rnn
    from oracle.tf32 import Tf32RNN

    torch.manual_seed(2)
    B, T, E, H = 128, 120, 256, 256
    ref = torch.nn.GRU(E, H, num_layers=2, batch_first=True)
    gru = b200rnn.from_torch(ref).to(DEV).eval()
    ln64 = torch.nn.LayerNorm(E).double()
    with torch.no_grad():
        ln64.weight.uniform_(0.5, 1.5)
        ln64.bias.uniform_(-0.2, 0.2)
    ln = torch.nn.LayerNorm(E).to(DEV)
    ln.load_state_dict(ln64.float().state_dict())
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, T, E, generator=g)
    wp = torch.randn(B, H, generator=g)
    xm = x.to(DEV).requires_grad_(True)
    with matmul_precision("tf32"):
        with torch.no_grad():
            pooled_ng = gru.forward_ln_sum(xm, ln)
        pooled = gru.forward_ln_sum(xm, ln)
    (pooled * wp.to(DEV)).sum().backward()
    torch.cuda.synchronize()

    # per-layer outputs of the kernels: layer 0 with the same LayerNorm prologue, layer 1 on its output
    from b200rnn.functional import rnn_forward_fused

    params = list(ref.parameters())
    g0, g1 = _one_layer("gru", params[:4], E, H, False), _one_layer("gru", params[4:], H, H, False)
    with matmul_precision("tf32"):
        y0 = rnn_forward_fused(xm.detach().transpose(0, 1), g0._flat_weights, g0._config(), None, ln.weight, ln.bias,
                               ln.eps)[0]
        y1 = rnn_forward_fused(y0, g1._flat_weights, g1._config())[0]
    x64 = x.double().requires_grad_(True)
    xln = ln64.double()(x64)
    orc = Tf32RNN("gru", [p.detach().double().numpy() for p in params], 2, False, rec_round=True)
    y = orc.forward(xln.detach().numpy().transpose(1, 0, 2), observed=[_np(y0), _np(y1)])[0]
    pooled_e = y.sum(axis=0)
    dxln, dps = orc.backward(np.broadcast_to(wp.double().numpy(), y.shape).copy())
    xln.backward(torch.from_numpy(dxln.transpose(1, 0, 2).copy()))
    # The one rounded operand the emulation cannot take from the kernels is LayerNorm(x): the prologue computes it in
    # fp32 and keeps it inside the library, so a few of its elements round to the other TF32 neighbour than the float64
    # LayerNorm does. What depends on the layer-0 projection's operands gets twice the usual gradient bound (1.4e-4 was
    # measured on an H100 for dx); everything downstream of layer 0's output keeps the usual one.
    errs = {"pooled_no_grad": _absmax(_np(pooled_ng), pooled_e), "pooled": _absmax(_np(pooled), pooled_e),
            "dx": _relmax(_np(xm.grad), x64.grad.numpy()), "dln_weight": _relmax(_np(ln.weight.grad),
                                                                                  ln64.weight.grad.numpy()),
            "dln_bias": _relmax(_np(ln.bias.grad), ln64.bias.grad.numpy())}
    for (n, _), p, d in zip(ref.named_parameters(), gru._flat_weights, dps):
        errs["d" + n] = _relmax(_np(p.grad), d)
    print("fused LayerNorm + time sum, TF32 vs emulation:", errs)
    for k, v in errs.items():
        tol = FEAT_TOL if k.startswith("pooled") else 2 * GRAD_RTOL if k in ("dx", "dln_weight", "dln_bias",
                                                                              "dweight_ih_l0") else GRAD_RTOL
        assert v <= tol, f"{k}: {v:.3e} > {tol:.0e} (all: {errs})"


def test_flag_reaches_the_kernels_and_ieee_restores_the_default_bitwise():
    import b200rnn

    torch.manual_seed(4)
    m = b200rnn.GRU(256, 256, num_layers=2, batch_first=True).to(DEV).eval()
    x = torch.randn(128, 50, 256, device=DEV)
    with torch.no_grad():
        y_default, h_default = m(x)
        with matmul_precision("tf32"):
            y_tf32, _ = m(x)
        with matmul_precision("ieee"):
            y_ieee, h_ieee = m(x)
    assert not torch.equal(y_tf32, y_default)
    assert (y_tf32 - y_default).abs().max().item() < 1e-2
    assert torch.equal(y_ieee, y_default) and torch.equal(h_ieee, h_default)


def test_streamed_and_serial_order_are_bitwise_equal_in_tf32_mode():
    """B = 128 streams its input projection into tc8, B = 160 runs it first (tests/test_gpu_streamed_projection.py);
    every batch row is computed by the same operations either way."""
    import b200rnn

    torch.manual_seed(5)
    m = b200rnn.GRU(256, 256, num_layers=2).to(DEV).eval()
    x = torch.randn(120, 160, 256, device=DEV)
    with torch.no_grad(), matmul_precision("tf32"):
        y_serial, h_serial = m(x)
        y_streamed, h_streamed = m(x[:, :128].contiguous())
    assert torch.equal(y_streamed, y_serial[:, :128])
    assert torch.equal(h_streamed, h_serial[:, :128])


def test_dropout_masks_of_forward_and_backward_agree_in_tf32_mode():
    """Train mode, p = 0.5, one step of one sequence: the units whose dW_ih_l1 column is zero are the ones the saved
    dropped layer-0 output zeroed. A forward of layer 1 alone on h0 * mask / (1 - p) reproduces the output (forward
    mask), and the input gradient matches the emulation through the same mask (backward mask)."""
    import b200rnn
    from oracle.tf32 import Tf32RNN

    p = 0.5
    torch.manual_seed(6)
    m = b200rnn.GRU(256, 256, num_layers=2, dropout=p).to(DEV).train()
    layer = [b200rnn.GRU(256, 256, num_layers=1).to(DEV).eval() for _ in range(2)]
    with torch.no_grad():
        for i, mod in enumerate(layer):
            for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                getattr(mod, n + "_l0").copy_(getattr(m, f"{n}_l{i}"))
    x = torch.randn(1, 1, 256, device=DEV, requires_grad=True)
    dy = torch.randn(1, 1, 256, device=DEV)
    with matmul_precision("tf32"):
        y, _ = m(x)
        (y * dy).sum().backward()
        with torch.no_grad():
            h0, _ = layer[0](x)
            kept = m.weight_ih_l1.grad.abs().sum(0) != 0
            y_check, _ = layer[1](h0 * kept / (1 - p))
    torch.cuda.synchronize()
    frac = 1.0 - kept.float().mean().item()
    assert 0.3 < frac < 0.7, frac
    assert (y - y_check).abs().max().item() <= 1e-6

    w = [p_.detach().double().cpu().numpy() for p_ in m._flat_weights]
    mask = kept.double().cpu().numpy() / (1 - p)
    e0, e1 = Tf32RNN("gru", w[:4], 1, False), Tf32RNN("gru", w[4:], 1, False)
    h0e = e0.forward(x.detach().double().cpu().numpy())[0]
    e1.forward(h0e * mask)
    dxin, _ = e1.backward(dy.double().cpu().numpy())
    dx, _ = e0.backward(dxin * mask)
    assert _relmax(_np(x.grad), dx) <= GRAD_RTOL


def test_captured_fuse_step_keeps_its_mode_and_matches_emulation():
    import b200rnn
    from oracle import ref_models
    from oracle.tf32 import Tf32RNN

    torch.manual_seed(7)
    args = dict(text_embed_size=1024, text_hidden_dims=128, rnn_layers=2, dropout=0.3, num_classes=2,
                audio_hidden_dims=256, audio_embed_size=256)
    ref = ref_models.RefFusion(**args).double().eval()
    m = b200rnn.fusion_net(**args)
    m.load_state_dict(ref.float().state_dict())
    ref.double()
    m = m.to(DEV).eval()
    for q in m.parameters():
        q.requires_grad = False
    m.fc_final[0].weight.requires_grad = True
    step = b200rnn.FusedFuseStep(m, exchange="none")
    B = 128
    g = torch.Generator().manual_seed(8)
    audio_c, text_c = torch.randn(B, 120, 256, generator=g), torch.randn(B, 30, 1024, generator=g)
    audio, text = audio_c.to(DEV), text_c.to(DEV)
    with matmul_precision("tf32"):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                step.features(b200rnn.FuseBatch(audio, text))
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_tf, static_af = step.features(b200rnn.FuseBatch(audio, text))
        graph.replay()
        torch.cuda.synchronize()
        tf1, af1 = static_tf.clone(), static_af.clone()
    w = m.fc_final[0].weight.detach()
    logits = torch.cat((tf1, af1), dim=1) @ w.t()

    with torch.no_grad():
        lstm = Tf32RNN("lstm", [p.numpy() for p in ref.lstm_net.parameters()], 2, True)
        out, hid, _ = lstm.forward(text_c.double().numpy().transpose(1, 0, 2))
        tf_e = ref.fc_out(ref_models._pool_with_attention(ref.attention_layer, torch.from_numpy(out).permute(1, 0, 2),
                                                          torch.from_numpy(hid).permute(1, 0, 2)))
        gru = Tf32RNN("gru", [p.numpy() for p in ref.lstm_net_audio.parameters()], 2, False, rec_round=True)
        y = gru.forward(ref.ln(audio_c.double()).numpy().transpose(1, 0, 2))[0]
        af_e = ref.fc_audio(torch.from_numpy(y.sum(axis=0)))
        logits_e = torch.cat((tf_e, af_e), dim=1) @ ref.fc_final[0].weight.t()
    err = (logits.double().cpu() - logits_e).abs().max().item()
    print(f"captured TF32 fuse step: logits vs emulation {err:.2e}")
    assert err <= FEAT_TOL

    with matmul_precision("ieee"):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(static_tf, tf1) and torch.equal(static_af, af1)
        tf_ieee, af_ieee = step.features(b200rnn.FuseBatch(audio, text))
        torch.cuda.synchronize()
    assert not torch.equal(af_ieee, af1)
