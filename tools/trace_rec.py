#!/usr/bin/env python
"""Debug: per-step, per-warp timeline (SM clock cycles) of the forward recurrence, CTA 0, lane 0 of each warp.
Needs the -DB200RNN_TRACE build:  make -C icassp2022-depression_b200 trace
    B200RNN_LIB=$PWD/icassp2022-depression_b200/lib_trace/libb200rnn.so python tools/trace_rec.py [gru|lstm|tc] [--json F]
gru / lstm: the FFMA kernel (rec_fwd_kernel). Stamps per (step, warp): 0 step top | 1-4 wait for chunk 0..3 passed |
5 butterfly done | 6 gates done | 7 exchange issued. The GRU runs at B = 96, which takes the 4-row FFMA config (bs4).
tc: the tensor-core GRU-256 body (rec_fwd_tc_body) at B = 128, T = 120, one layer, x-projection streamed, run twice:
the fp16-pair kernel (no-grad GRU.forward_ln_sum -> b200rnn_forward_fused) and the 3xTF32 kernel (module forward).
Stamps per (step, warp), 16 per row: 0 step top | 1 own-slice wait passed | 2-4 peer-slice waits passed | 5 contraction
done | 6 k-half swap done | 7 update done | 8 slice sent | 9 GiReady passed | 10 load_gi issued. A stamp the body does not
write stays 0. Printed per phase: the median over steps 8 .. T-8 of the cycles since the previous stamp, averaged over
the 8 warps; `step` is top to next top. --json F also writes them with the card, power limit and clocks."""
import ctypes, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))
import torch, b200rnn
from b200rnn import _lib
lib = _lib.load()
lib.b200rnn_debug_set_trace.argtypes = [ctypes.c_void_p]
args = [a for a in sys.argv[1:] if not a.startswith("--")]
kind = args[0] if args else "gru"
json_out = sys.argv[sys.argv.index("--json") + 1] if "--json" in sys.argv else None
if json_out in args:
    args.remove(json_out)
dev = torch.device("cuda:0")

TC_PHASES = ["own wait", "peer 1", "peer 2", "peer 3", "contraction tail", "k-half swap", "update", "send",
             "GiReady", "load_gi"]


def traced(run, T, width):
    with torch.no_grad():
        run()
        torch.cuda.synchronize()
        buf = torch.zeros(T, 8, width, dtype=torch.int64, device=dev)
        lib.b200rnn_debug_set_trace(buf.data_ptr())
        run()
        torch.cuda.synchronize()
        lib.b200rnn_debug_set_trace(None)
    return buf.cpu()


def tc_phases(t):
    """median over the middle steps of each phase's cycles since the previous stamp the body writes (a phase whose stamp
    it does not write is absent), to the next step's top for the last one; mean over the warps"""
    T = t.shape[0]
    steps = range(8, T - 8)
    present = [k for k in range(1, 11) if bool(t[8:T - 8, :, k].any())]
    out = {}
    prev = 0
    for k in present + [11]:
        name = TC_PHASES[k - 1] if k <= 10 else "to next step top"
        vals = []
        for w in range(8):
            d = []
            for s in steps:
                end = int(t[s + 1, w, 0]) if k == 11 else int(t[s, w, k])
                d.append(end - int(t[s, w, prev]))
            d.sort()
            vals.append(d[len(d) // 2])
        out[name] = sum(vals) / len(vals)
        prev = k
    st = []
    for w in range(8):
        d = sorted(int(t[s + 1, w, 0]) - int(t[s, w, 0]) for s in steps)
        st.append(d[len(d) // 2])
    out["step"] = sum(st) / len(st)
    return out


if kind == "tc":
    T, B = 120, 128
    torch.manual_seed(0)
    m = b200rnn.GRU(256, 256, num_layers=1, batch_first=True).to(dev).eval()
    ln = torch.nn.LayerNorm(256).to(dev)
    x = torch.randn(B, T, 256, device=dev)
    result = {"shape": {"B": B, "T": T, "H": 256, "layers": 1, "streamed_xproj": True}, "cycles_per_phase": {}}
    for name, run in (("h16 (forward_ln_sum, fp16 pairs)", lambda: m.forward_ln_sum(x, ln)),
                      ("x3 (module forward, 3xTF32)", lambda: m(x))):
        ph = tc_phases(traced(run, T, 16))
        result["cycles_per_phase"][name] = ph
        print(f"{name}: step {ph['step']:.0f} cycles")
        for k, v in ph.items():
            if k != "step":
                print(f"  {k:>18s} {v:7.0f}  ({100 * v / ph['step']:4.1f} %)")
    if json_out:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
        result["gpu"] = q
        result["how"] = ("tools/trace_rec.py tc on the -DB200RNN_TRACE build: CTA 0, lane 0 of each of the 8 compute "
                         "warps; per phase the median over steps 8 .. T-8 of the clock64 cycles since the previous "
                         "stamp, averaged over the warps. Stamping perturbs the schedule; compare builds, not absolutes.")
        with open(json_out, "w") as f:
            json.dump(result, f, indent=1)
    sys.exit(0)

if kind == "gru":
    m = b200rnn.GRU(256, 256, num_layers=1, batch_first=True).to(dev).eval(); x = torch.randn(96, 120, 256, device=dev); T = 120; nch = 4
else:
    m = b200rnn.LSTM(1024, 128, num_layers=1, bidirectional=True).to(dev).eval(); x = torch.randn(30, 128, 1024, device=dev); T = 30; nch = 2
t = traced(lambda: m(x), T, 8)
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
