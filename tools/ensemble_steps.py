#!/usr/bin/env python
"""What running M models in one call saves: torch.func.vmap over stacked b200rnn modules (b200rnn/func.py: one
recurrence launch per layer for all models) against a Python loop of M eager b200rnn calls and against a loop of M stock
cuDNN modules.

Workloads, fp32, default (3xTF32) precision; cuDNN with its RNN math in IEEE fp32
(torch.backends.cudnn.rnn.fp32_precision = "ieee"):
  * audio_gru256: GRU(256, 256, num_layers=2), batch_first (the audio branch);
  * text_bilstm128: LSTM(1024, 128, num_layers=2, bidirectional) (the text branch);
  * lstm512: LSTM(256, 512, num_layers=2).
Shapes: the EATD batch (B = 8, T = 3) and B = 64, T = 120; M in {1, 3, 8, 32}. Per call: the forward under no_grad, and
forward + backward (loss = sum of squares of the output, autograd outside vmap). Per-sample gradients: 32 samples of
one sequence each (T = 3 and T = 120), vmap(grad(loss), in_dims=(None, 0)) against a loop of 32 eager backward calls.
Every variant is timed with CUDA events around `reps` calls (fewer where they would pass 200 ms, at least one) after a
warm-up call, in alternation, `rounds` times; the JSON (rewritten after every row) keeps every round and the largest difference between the ensemble's output and the loop's. The card name, its power
limit and clocks are read in the same run.

    python tools/ensemble_steps.py [--reps 10] [--rounds 3] [--out tools/ensemble_steps_results.json]
"""
import argparse
import copy
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))

import torch  # noqa: E402
from torch.func import functional_call, grad, stack_module_state, vmap  # noqa: E402

import b200rnn  # noqa: E402

WORKLOADS = {
    "audio_gru256": dict(kind="gru", I=256, H=256, L=2, bi=False, bf=True),
    "text_bilstm128": dict(kind="lstm", I=1024, H=128, L=2, bi=True, bf=False),
    "lstm512": dict(kind="lstm", I=256, H=512, L=2, bi=False, bf=False),
}
MS = (1, 3, 8, 32)
SHAPES = ((8, 3), (64, 120))
PER_SAMPLE_N, PER_SAMPLE_TS = 32, (3, 120)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 else None
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn, reps, budget_ms=200.0):
    """ms per call over `reps` calls after one warm-up call; fewer calls (at least one) where `reps` of them would
    take longer than budget_ms"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    reps = max(1, min(reps, int(budget_ms / max(e0.elapsed_time(e1), 1e-3))))
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def save(res, path):
    with open(path, "w") as f:
        json.dump(res, f, indent=1)


def make(w, M, stock=False):
    ns = torch.nn if stock else b200rnn
    ctor = ns.GRU if w["kind"] == "gru" else ns.LSTM
    return [ctor(w["I"], w["H"], num_layers=w["L"], bidirectional=w["bi"], batch_first=w["bf"]).cuda()
            for _ in range(M)]


def ensemble_variants(w, M, B, T):
    models = make(w, M)
    stock = make(w, M, stock=True)
    for s, m in zip(stock, models):
        s.load_state_dict(m.state_dict())
    params, bufs = stack_module_state(models)
    base = copy.deepcopy(models[0])
    shape = (M, B, T, w["I"]) if w["bf"] else (M, T, B, w["I"])
    x = torch.randn(shape, device="cuda")
    f = vmap(lambda p, b, xx: functional_call(base, (p, b), (xx,))[0])

    def vmap_fwd():
        with torch.no_grad():
            f(params, bufs, x)

    def vmap_fwd_bwd():
        f(params, bufs, x).square().sum().backward()

    def loop(ms, train):
        def run():
            for m, model in enumerate(ms):
                if train:
                    model(x[m])[0].square().sum().backward()
                else:
                    with torch.no_grad():
                        model(x[m])
        return run

    with torch.no_grad():
        diff = max((f(params, bufs, x)[m] - models[m](x[m])[0]).abs().max().item() for m in range(M))
    return {"vmap_fwd": vmap_fwd, "vmap_fwd_bwd": vmap_fwd_bwd, "loop_fwd": loop(models, False),
            "loop_fwd_bwd": loop(models, True), "cudnn_loop_fwd": loop(stock, False),
            "cudnn_loop_fwd_bwd": loop(stock, True)}, diff


def per_sample_variants(w, T):
    model = make(w, 1)[0]
    params = {n: p.detach() for n, p in model.named_parameters()}
    bufs = dict(model.named_buffers())
    N, bdim = PER_SAMPLE_N, 0 if w["bf"] else 1
    xs = torch.randn(N, T, w["I"], device="cuda")

    def loss(p, xx):
        return functional_call(model, (p, bufs), (xx.unsqueeze(bdim),))[0].square().sum()

    g = vmap(grad(loss), in_dims=(None, 0))

    def vmapped():
        g(params, xs)

    def loop():
        for n in range(N):
            model.zero_grad(set_to_none=True)
            model(xs[n].unsqueeze(bdim))[0].square().sum().backward()

    return {"vmap_grad": vmapped, "per_sample_loop": loop}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "ensemble_steps_results.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ensemble_steps.py needs a CUDA device")
    torch.backends.cudnn.rnn.fp32_precision = "ieee"
    res = {"gpu": gpu_info(), "torch": torch.__version__, "reps": args.reps, "rounds": args.rounds,
           "ensembles": [], "per_sample": []}
    for name, w in WORKLOADS.items():
        for B, T in SHAPES:
            for M in MS:
                fns, diff = ensemble_variants(w, M, B, T)
                rounds = {k: [] for k in fns}
                for _ in range(args.rounds):
                    for k, fn in fns.items():
                        rounds[k].append(timed(fn, args.reps))
                row = {"workload": name, "M": M, "B": B, "T": T, "ms_per_call": rounds,
                       "max_abs_diff_vmap_vs_loop": diff}
                res["ensembles"].append(row)
                print(name, M, B, T, {k: round(min(v), 3) for k, v in rounds.items()}, "diff", diff, flush=True)
                save(res, args.out)
                del fns
                torch.cuda.empty_cache()
        for T in PER_SAMPLE_TS:
            fns = per_sample_variants(w, T)
            rounds = {k: [] for k in fns}
            for _ in range(args.rounds):
                for k, fn in fns.items():
                    rounds[k].append(timed(fn, args.reps))
            res["per_sample"].append({"workload": name, "N": PER_SAMPLE_N, "T": T, "ms_per_call": rounds})
            print(name, "per-sample", T, {k: round(min(v), 3) for k, v in rounds.items()}, flush=True)
            save(res, args.out)
    res["gpu_after"] = gpu_info()
    save(res, args.out)


if __name__ == "__main__":
    main()
