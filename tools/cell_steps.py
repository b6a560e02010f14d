#!/usr/bin/env python
"""What one recurrent step costs through three paths, for a user who steps a model frame by frame or writes a custom loop:

  * `b200rnn_cell`: b200rnn.GRUCell / LSTMCell (one fused launch per forward step);
  * `torch_cell`:   stock torch.nn.GRUCell / LSTMCell(...).cuda() (cuBLAS GEMMs and torch's fused pointwise cell; torch's
                    default fp32 matmul precision, i.e. no TF32);
  * `b200rnn_seq`:  b200rnn.GRU / LSTM (1 layer) called with T = 1 and hx, the sequence machinery for one step.

All three run in fp32 with the same weights. Per (cell, I, H, B) and pass (`fwd`: forward under no_grad; `fwd_bwd`: the
forward with the weights requiring grad, then backward of the sum of the last state), a loop of T = 120 steps is timed
  * `eager`: as Python runs it, CUDA events around the loop;
  * `graph`: the same loop captured once in a CUDA graph, events around one replay.
Rounds alternate the three paths in one process; the result is the median over rounds, in microseconds per step.

    python tools/cell_steps.py [--rounds 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))

import torch  # noqa: E402

import b200rnn  # noqa: E402

T = 120
SHAPES = ((256, 256), (1024, 128))
BATCHES = (1, 8, 128, 1024)
PATHS = ("b200rnn_cell", "torch_cell", "b200rnn_seq")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 else None
    except (OSError, subprocess.SubprocessError):
        return None


def make_loops(kind, I, H, B, dev, train):
    """{path: loop()} where loop() runs T steps from a zero state (and the backward with `train`)"""
    torch.manual_seed(0)
    stock = (torch.nn.GRUCell if kind == "gru" else torch.nn.LSTMCell)(I, H)
    mine = b200rnn.from_torch(stock).to(dev)
    torch_cell = stock.to(dev)
    seq = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(I, H).to(dev)
    with torch.no_grad():
        for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
            getattr(seq, f"{n}_l0").copy_(getattr(stock, n))
    for m in (mine, torch_cell, seq):
        m.requires_grad_(train)
    xs = torch.randn(T, B, I, device=dev)
    zero = torch.zeros(B, H, device=dev)

    def cell_loop(cell):
        def loop():
            state = zero if kind == "gru" else (zero, zero)
            for t in range(T):
                state = cell(xs[t], state)
            last = state if kind == "gru" else state[0]
            if train:
                last.sum().backward()
        return loop

    def seq_loop():
        state = zero[None] if kind == "gru" else (zero[None], zero[None])
        for t in range(T):
            _, state = seq(xs[t:t + 1], state)
        last = state if kind == "gru" else state[0]
        if train:
            last.sum().backward()

    return {"b200rnn_cell": cell_loop(mine), "torch_cell": cell_loop(torch_cell), "b200rnn_seq": seq_loop}, \
        (mine, torch_cell, seq)


def time_call(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / T  # us per step


def measure(kind, I, H, B, dev, train, rounds):
    loops, modules = make_loops(kind, I, H, B, dev, train)
    ctx = torch.enable_grad if train else torch.no_grad
    res = {}
    with ctx():
        for fn in loops.values():  # warm-up: module loads, cuBLAS heuristics, the caching allocator
            fn()
            fn()
        torch.cuda.synchronize()
        eager = {p: [] for p in PATHS}
        for _ in range(rounds):
            for p in PATHS:
                eager[p].append(time_call(loops[p]))
        graphs = {}
        for p in PATHS:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                loops[p]()
            torch.cuda.current_stream().wait_stream(side)
            for m in modules:
                m.zero_grad(set_to_none=True)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                loops[p]()
            graphs[p] = g
        for g in graphs.values():
            g.replay()
        torch.cuda.synchronize()
        graph = {p: [] for p in PATHS}
        for _ in range(rounds):
            for p in PATHS:
                graph[p].append(time_call(graphs[p].replay))
        del graphs
    for p in PATHS:
        res[p] = {"eager_us_per_step": statistics.median(eager[p]), "graph_us_per_step": statistics.median(graph[p])}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "cell_steps.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.fp32_precision = "ieee"  # fp32 everywhere: 3xTF32 in b200rnn, no TF32 in cuBLAS
    out = {"device": torch.cuda.get_device_name(dev), "nvidia_smi (name, power.limit, clocks.sm, clocks.max.sm)":
           gpu_info(), "T": T, "rounds": args.rounds, "unit": "us per step, median over rounds", "results": {}}
    for kind in ("gru", "lstm"):
        for I, H in SHAPES:
            for B in BATCHES:
                key = f"{kind}_I{I}_H{H}_B{B}"
                out["results"][key] = {
                    "fwd": measure(kind, I, H, B, dev, False, args.rounds),
                    "fwd_bwd": measure(kind, I, H, B, dev, True, args.rounds),
                }
                torch.cuda.empty_cache()
                print(key, json.dumps(out["results"][key]), flush=True)
    text = json.dumps(out, indent=1)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
