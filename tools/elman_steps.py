#!/usr/bin/env python
"""What the Elman recurrence (the Elman kernels of csrc/rnn_anyh.cu) and the RNNCell kernels cost, against stock
cuDNN / ATen.

Sequence: one unidirectional layer, time-major, T = 120, I = 64, H in {64, 128, 256, 512, 1024}, B in {16, 64, 128},
nonlinearity tanh and relu:
  * `ours`: b200rnn.RNN: the forward and backward recurrence launches alone (the library's profile hook: event pairs
    around each launch), the whole forward + backward of the module (CUDA events around `reps` calls), and the config
    the library chose (B200RNN_DEBUG line, read from a subprocess: cluster width C, batch rows BS, weight tier);
  * `cudnn_fp32` / `cudnn_tf32`: stock torch.nn.RNN(...).cuda() with cuDNN's RNN math in IEEE fp32
    (torch.backends.cudnn.rnn.fp32_precision = "ieee") and in TF32 ("tf32"): forward alone and forward + backward.
Cells: RNNCell(I = H, H) for H in {64, 256, 1024}, B in {1, 128}: a loop of `steps` forward steps (h fed back), captured
once in a CUDA graph, events around a replay; b200rnn.RNNCell against torch.nn.RNNCell in IEEE fp32.
Everything is timed in alternation, `rounds` times, after a warm-up; the JSON keeps every round. The card name, its
power limit and clocks are read in the same run.

    python tools/elman_steps.py [--reps 10] [--rounds 3] [--out tools/elman_steps_results.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))

import torch  # noqa: E402

import b200rnn  # noqa: E402
from b200rnn import _lib  # noqa: E402

HS = (64, 128, 256, 512, 1024)
BS = (16, 64, 128)
NONLIN = ("tanh", "relu")
T, I = 120, 64
CELL_HS, CELL_BS, CELL_STEPS = (64, 256, 1024), (1, 128), 50


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 else None
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _loss(out):
    return out[0].square().sum() + out[1].sum()


def ours(model, x, reps):
    def step():
        _loss(model(x)).backward()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    step_ms = timed(step, reps)
    _lib.profile(True)
    for _ in range(reps):
        step()
    torch.cuda.synchronize()
    fwd_ms, fwd_n = _lib.profile_read(_lib.PROF_REC_FWD)
    bwd_ms, bwd_n = _lib.profile_read(_lib.PROF_REC_BWD)
    _lib.profile(False)
    return {"rec_fwd_ms_per_launch": fwd_ms / max(fwd_n, 1), "rec_bwd_ms_per_launch": bwd_ms / max(bwd_n, 1),
            "fwd_bwd_ms": step_ms}


def cudnn(model, x, reps, precision):
    saved = torch.backends.cudnn.rnn.fp32_precision
    torch.backends.cudnn.rnn.fp32_precision = precision
    try:
        def fwd():
            with torch.no_grad():
                model(x)

        def step():
            _loss(model(x)).backward()

        for _ in range(2):
            fwd()
            step()
        torch.cuda.synchronize()
        return {"fwd_ms": timed(fwd, reps), "fwd_bwd_ms": timed(step, reps)}
    finally:
        torch.backends.cudnn.rnn.fp32_precision = saved


def cell_graph_us(cell, x, h0):
    """us per step of CELL_STEPS forward steps (h fed back), captured in one CUDA graph"""
    def loop():
        h = h0
        for _ in range(CELL_STEPS):
            h = cell(x, h)
        return h

    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            loop()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            loop()
    g.replay()
    torch.cuda.synchronize()
    return 1e3 * timed(g.replay, 20) / CELL_STEPS


_CFG = r"""
import sys, torch, b200rnn
T, I = int(sys.argv[1]), int(sys.argv[2])
for spec in sys.argv[3:]:
    nl, H, B = spec.split(":")
    print("SHAPE", spec, file=sys.stderr, flush=True)
    m = b200rnn.RNN(I, int(H), nonlinearity=nl).cuda()
    x = torch.randn(T, int(B), I, device="cuda", requires_grad=True)
    m(x)[0].sum().backward()
    torch.cuda.synchronize()
"""


def chosen_configs(specs):
    """{"nl:H:B": [the B200RNN_DEBUG config lines of one forward + backward]}, from one subprocess"""
    env = dict(os.environ, B200RNN_DEBUG="1")
    r = subprocess.run([sys.executable, "-c", _CFG, str(T), str(I), *specs], capture_output=True, text=True, env=env,
                       cwd=os.path.join(ROOT, "icassp2022-depression_b200"), timeout=600)
    out, cur = {}, None
    for ln in r.stderr.splitlines():
        if ln.startswith("SHAPE "):
            cur = ln.split()[1]
            out[cur] = []
        elif cur and re.search(r"(fwd|bwd) elman cfg", ln):
            out[cur].append(ln)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "elman_steps.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    out = {"device": torch.cuda.get_device_name(dev), "nvidia_smi": gpu_info(),
           "library": os.path.relpath(_lib.LIB_PATH, ROOT), "T": T, "I": I, "bidirectional": False, "num_layers": 1,
           "reps": args.reps, "cudnn": "torch.nn.RNN(...).cuda(); cudnn_fp32: rnn.fp32_precision='ieee', "
           "cudnn_tf32: 'tf32'", "shapes": [], "cells": []}
    configs = chosen_configs([f"{nl}:{H}:{B}" for nl in NONLIN for H in HS for B in BS])
    for nl in NONLIN:
        for H in HS:
            for B in BS:
                torch.manual_seed(0)
                x = torch.randn(T, B, I, device=dev, requires_grad=True)
                mine = b200rnn.RNN(I, H, nonlinearity=nl).to(dev)
                ref = b200rnn.modules._TORCH_RNN(I, H, nonlinearity=nl).to(dev)
                res = {"nonlinearity": nl, "H": H, "B": B, "config": configs.get(f"{nl}:{H}:{B}"),
                       "rounds": {"ours": [], "cudnn_fp32": [], "cudnn_tf32": []}}
                for _ in range(args.rounds):
                    res["rounds"]["ours"].append(ours(mine, x, args.reps))
                    res["rounds"]["cudnn_fp32"].append(cudnn(ref, x, args.reps, "ieee"))
                    res["rounds"]["cudnn_tf32"].append(cudnn(ref, x, args.reps, "tf32"))
                out["shapes"].append(res)
                print(json.dumps(res), flush=True)
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    try:
        for H in CELL_HS:
            for B in CELL_BS:
                torch.manual_seed(0)
                ref = torch.nn.RNNCell(H, H).to(dev)
                mine = b200rnn.from_torch(ref).to(dev)
                x, h0 = torch.randn(B, H, device=dev), torch.randn(B, H, device=dev)
                res = {"cell": "RNNCell", "I": H, "H": H, "B": B, "steps_per_graph": CELL_STEPS,
                       "rounds": {"ours_graph_us_per_step": [], "torch_graph_us_per_step": []}}
                for _ in range(args.rounds):
                    res["rounds"]["ours_graph_us_per_step"].append(cell_graph_us(mine, x, h0))
                    res["rounds"]["torch_graph_us_per_step"].append(cell_graph_us(ref, x, h0))
                out["cells"].append(res)
                print(json.dumps(res), flush=True)
    finally:
        torch.backends.cuda.matmul.fp32_precision = saved
    text = json.dumps(out, indent=1)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
