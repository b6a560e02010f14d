"""Milliseconds per call, forward and forward + backward, of an fp32 module under ``torch.autocast("cuda",
dtype=float16)`` (the 16-bit kernels on fp32 master parameters), of the same module without autocast, of its 16-bit twin
(``copy.deepcopy(m).half()``) and of stock cuDNN (``torch.nn.GRU`` / ``LSTM``) under the same autocast region.

Shapes: the audio GRU-256 (B = 128, T = 120, 2 layers), the text BiLSTM H = 128 and 256 (B = 64, T = 30, 1024-d input,
2 layers), an LSTM-512 at B = 16 and a GRU-720 at B = 128 (T = 120). Each round times ``--iters`` calls of every variant
with CUDA events, the variants alternated; the result is the median over ``--rounds`` rounds. The card's name and power
limit are read in the same run. Writes tools/autocast_steps_results.json unless ``--out`` says otherwise.

    python tools/autocast_steps.py [--rounds 7] [--iters 20] [--out PATH]
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))

import torch  # noqa: E402

import b200rnn  # noqa: E402
from b200rnn.modules import _TORCH_GRU, _TORCH_LSTM  # noqa: E402

SHAPES = [
    # name, kind, input size, hidden size, layers, bidirectional, B, T
    ("audio_gru256", "gru", 256, 256, 2, False, 128, 120),
    ("text_bilstm128", "lstm", 1024, 128, 2, True, 64, 30),
    ("text_bilstm256", "lstm", 1024, 256, 2, True, 64, 30),
    ("lstm512_b16", "lstm", 512, 512, 1, False, 16, 120),
    ("gru720_b128", "gru", 720, 720, 1, False, 128, 120),
]


def _time(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def measure(shape, rounds, iters, dev):
    name, kind, I, H, L, bi, B, T = shape
    torch.manual_seed(0)
    ours = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(I, H, num_layers=L, bidirectional=bi).to(dev).train()
    twin = copy.deepcopy(ours).half()
    stock = (_TORCH_GRU if kind == "gru" else _TORCH_LSTM)(I, H, num_layers=L, bidirectional=bi).to(dev).train()
    x32 = torch.randn(T, B, I, device=dev, requires_grad=True)
    x16 = x32.detach().half().requires_grad_(True)
    variants = {"fp32_autocast": (ours, x32, True), "fp32": (ours, x32, False), "f16_twin": (twin, x16, False),
                "cudnn_autocast": (stock, x32, True)}

    def fwd(m, x, amp):
        def run():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                m(x)
        return run

    def fwd_bwd(m, x, amp):
        def run():
            with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                y = m(x)[0]
            y.float().sum().backward()
        return run

    fns = {(v, p): (fwd if p == "fwd" else fwd_bwd)(*variants[v]) for v in variants for p in ("fwd", "fwd_bwd")}
    for fn in fns.values():   # warm every path and the allocator
        fn()
        fn()
    torch.cuda.synchronize()
    samples = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            samples[k].append(_time(fn, iters))
    out = {"shape": dict(kind=kind, input_size=I, hidden_size=H, num_layers=L, bidirectional=bi, batch=B, seq_len=T)}
    for v in variants:
        f = statistics.median(samples[(v, "fwd")])
        fb = statistics.median(samples[(v, "fwd_bwd")])
        out[v] = {"fwd_ms": round(f, 4), "fwd_bwd_ms": round(fb, 4), "bwd_ms": round(fb - f, 4)}
    return name, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "autocast_steps_results.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("autocast_steps.py needs a CUDA device")
    dev = torch.device("cuda")
    res = {"card": _card(), "rounds": args.rounds, "iters": args.iters,
           "note": "median ms per call over alternated rounds; bwd_ms = fwd_bwd_ms - fwd_ms (the forward of fwd_bwd "
                   "saves for backward, so this is approximate)", "results": {}}
    for shape in SHAPES:
        name, r = measure(shape, args.rounds, args.iters, dev)
        res["results"][name] = r
        print(name, json.dumps(r), flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("card:", res["card"])


if __name__ == "__main__":
    main()
