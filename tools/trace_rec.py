#!/usr/bin/env python
"""Debug: per-step, per-warp timeline (SM clock cycles) of the forward recurrence, CTA 0, lane 0 of each warp.
Needs the -DB200RNN_TRACE build:  make -C icassp2022-depression_b200 trace
    B200RNN_LIB=$PWD/icassp2022-depression_b200/lib_trace/libb200rnn.so python tools/trace_rec.py [gru|lstm]
Stamps per (step, warp): 0 step top | 1-4 wait for chunk 0..3 passed | 5 butterfly done | 6 gates done | 7 exchange issued.
The GRU runs at B = 96, which takes the 4-row FFMA config (bs4); the tensor-core config (B > 120) has no stamps."""
import ctypes, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))
import torch, b200rnn
from b200rnn import _lib
lib = _lib.load()
lib.b200rnn_debug_set_trace.argtypes = [ctypes.c_void_p]
kind = sys.argv[1] if len(sys.argv) > 1 else "gru"
dev = torch.device("cuda:0")
if kind == "gru":
    m = b200rnn.GRU(256, 256, num_layers=1, batch_first=True).to(dev).eval(); x = torch.randn(96, 120, 256, device=dev); T = 120; nch = 4
else:
    m = b200rnn.LSTM(1024, 128, num_layers=1, bidirectional=True).to(dev).eval(); x = torch.randn(30, 128, 1024, device=dev); T = 30; nch = 2
with torch.no_grad():
    m(x)
    buf = torch.zeros(T, 8, 8, dtype=torch.int64, device=dev)
    lib.b200rnn_debug_set_trace(buf.data_ptr())
    m(x)
    torch.cuda.synchronize()
    lib.b200rnn_debug_set_trace(None)
t = buf.cpu()
for s in (10, 11):
    base = int(t[s, :, 0].min())
    print(f"step {s}: (cycles relative to the earliest warp's step top; next step's earliest top at {int(t[s + 1, :, 0].min()) - base})")
    for w in range(8):
        r = t[s, w]
        if int(r[0]) == 0:
            continue
        waits = "/".join(str(int(r[1 + c]) - base) for c in range(nch))
        print(f"  warp {w}: top {int(r[0]) - base:5d}  waits passed {waits:>24s}  butterfly done {int(r[5]) - base:5d}  "
              f"gates {int(r[6]) - base:5d}  sent {int(r[7]) - base:5d}")
