#!/usr/bin/env python
"""Small shapes through every recurrence variant, for compute-sanitizer (memcheck / racecheck):
    compute-sanitizer --tool memcheck python tools/sanitize_paths.py
    compute-sanitizer --tool memcheck python tools/sanitize_paths.py rnn   # recurrence only
The GRU H=256 layer also runs at B = 96, which needs the 4-row clusters (bs4: the 2-row ones do not all fit at once).
    compute-sanitizer --tool memcheck python tools/sanitize_paths.py cells # GRUCell / LSTMCell forward + backward only
    compute-sanitizer --tool memcheck python tools/sanitize_paths.py strided # caller-laid-out x / dy / y / dx
    compute-sanitizer --tool racecheck python tools/sanitize_paths.py anyh # runtime-sized recurrence (rnn_anyh.cu) only:
        GRU H = 192 (W_hh in shared memory) and LSTM H = 768 (W_hh from L2), fixed-length and ragged, with hx and dh_0
"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))
import torch, b200rnn
from torch.nn.utils.rnn import pack_padded_sequence
dev = torch.device("cuda:0")
torch.manual_seed(0)
if sys.argv[1:] == ["anyh"]:
    # B = 5 on clusters planned for more rows: idle threads past the batch, a partial last warp, unequal slices at 464
    for kind, I, H, B, T in (("gru", 24, 192, 5, 4), ("lstm", 24, 768, 5, 3), ("lstm", 24, 464, 3, 3)):
        m = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(I, H, bidirectional=True).to(dev)
        x = torch.randn(T, B, I, device=dev, requires_grad=True)
        h0 = torch.randn(2, B, H, device=dev, requires_grad=True)
        hx = h0 if kind == "gru" else (h0, torch.randn(2, B, H, device=dev))
        out = m(x, hx)
        (out[0].sum() + (out[1] if kind == "gru" else out[1][0]).sum()).backward()
        xp = pack_padded_sequence(x.detach().requires_grad_(True), torch.tensor([3, 1, 2, 3, 2][:B]),
                                  enforce_sorted=False)
        m(xp)[0].data.sum().backward()
        torch.cuda.synchronize()
        print(kind, H, "ok", flush=True)
    sys.exit(0)
if sys.argv[1:] == ["strided"]:
    # the whole layout matrix of tests/test_gpu_strided_io.py (offset, gapped, broadcast and size-1 x, dy, y and dx;
    # both batch_first settings, the _hx and _fused C ABI pairs, autocast, hx, ragged, the LayerNorm fold), in this
    # process; test_routes only re-runs the catalogue's forwards in a child process to read their debug lines
    import pytest
    sys.exit(pytest.main(["-q", "-p", "no:cacheprovider", "-x", os.path.join(ROOT, "tests", "test_gpu_strided_io.py"),
                          "-k", "not test_routes"]))
if sys.argv[1:] == ["cells"]:
    # K and batch tails, unaligned rows (odd offsets into larger buffers), no bias, no state, both contractions
    for kind, I, H, B, bias in (("gru", 3, 5, 7, True), ("lstm", 257, 129, 9, False), ("gru", 256, 256, 130, False),
                                ("lstm", 40, 100, 33, True)):
        cell = (b200rnn.GRUCell if kind == "gru" else b200rnn.LSTMCell)(I, H, bias=bias).to(dev)
        x = torch.randn(B * I + 1, device=dev)[1:].view(B, I).requires_grad_(True)
        h = torch.randn(B * H + 1, device=dev)[1:].view(B, H).requires_grad_(True)
        for prec in ("ieee", "tf32"):
            torch.backends.cuda.matmul.fp32_precision = prec
            for hx in (None, h if kind == "gru" else (h, torch.randn(B, H, device=dev))):
                out = cell(x, hx)
                (out if kind == "gru" else out[0] + out[1]).sum().backward()
        torch.cuda.synchronize()
        print(kind, I, H, B, "ok", flush=True)
    sys.exit(0)
for kind, I, H, L, bi in (("gru", 64, 256, 2, False), ("lstm", 64, 128, 2, True), ("gru", 32, 128, 1, True), ("lstm", 32, 256, 1, False)):
    cls = b200rnn.GRU if kind == "gru" else b200rnn.LSTM
    m = cls(I, H, num_layers=L, bidirectional=bi, batch_first=True, dropout=0.3 if L > 1 else 0.0).to(dev).train()
    T = 6
    for B in (9, 96) if (kind, H) == ("gru", 256) else (9,):
        x = torch.randn(B, T, I, device=dev, requires_grad=True)
        y = m.train()(x)[0]
        y.sum().backward()
        lengths = torch.tensor([6, 1, 3, 6, 2, 5, 4, 6, 1] * (B // 9) + [6] * (B % 9))
        xp = pack_padded_sequence(x.detach().requires_grad_(True), lengths, batch_first=True, enforce_sorted=False)
        yp = m(xp)[0]
        yp.data.sum().backward()
        with torch.no_grad():
            m.eval()(x)
        torch.cuda.synchronize()
        print(kind, H, B, "ok", flush=True)
if sys.argv[1:] == ["rnn"]:
    sys.exit(0)
# round 2: the fused shells (LayerNorm prologue + pooled gradient under autograd, attention pooling fwd/bwd, Softmax+CE,
# MN-major wgrad GEMMs, the single-launch fuse head with Adam)
cfg = dict(num_classes=2, dropout=0.3, rnn_layers=2, embedding_size=256, hidden_dims=128)
am = b200rnn.AudioBiLSTM(cfg).to(dev).train()
xa = torch.randn(5, 7, 256, device=dev, requires_grad=True)
p, loss = b200rnn.softmax_cross_entropy(am.forward_logits(xa), torch.randint(0, 2, (5,), device=dev))
loss.backward()
tm = b200rnn.TextBiLSTM(dict(num_classes=2, dropout=0.3, rnn_layers=2, embedding_size=128, hidden_dims=128)).to(dev).train()
xt = torch.randn(5, 6, 128, device=dev, requires_grad=True)
tm(xt).sum().backward()
fm = b200rnn.fusion_net(128, 128, 2, 0.3, 2, 128, 128).to(dev).train()
for q in fm.parameters():
    q.requires_grad = False
fm.fc_final[0].weight.requires_grad = True
st = b200rnn.FusedFuseStep(fm, lr=1e-3)
for _ in range(2):
    st(b200rnn.FuseBatch(torch.randn(6, 5, 128, device=dev), torch.randn(6, 4, 128, device=dev)),
       torch.randint(0, 2, (6,), device=dev))
torch.cuda.synchronize()
print("sanitize_paths done")
