#!/usr/bin/env python
"""What a Jacobian-vector product through the sequence modules costs: b200rnn's forward alone and torch.func.jvp
(b200rnn_forward_tangent: the tangent GEMMs and one tangent recurrence launch per layer) against stock torch.nn's jvp on
the GPU with cuDNN disabled, and what stock does with cuDNN enabled (a time, or the error it raises); then jacfwd-style
vmap(jvp) over M = 8 / 32 tangent directions of x against a loop of M jvp calls.

Workloads, fp32, eval mode, default (3xTF32) precision, tangent w.r.t. x only:
  * audio_gru256_b64 / _b128: GRU(256, 256, num_layers=2), batch_first, B = 64 / 128, T = 120 (the audio branch);
  * text_bilstm128: LSTM(1024, 128, num_layers=2, bidirectional), B = 64, T = 30 (the text branch);
  * lstm512: LSTM(512, 512), B = 16, T = 120;
  * rnn_tanh256: RNN(256, 256, nonlinearity='tanh'), B = 64, T = 120.
Each variant is timed with CUDA events around `reps` calls (a window of tens of ms at the small shapes) after a
warm-up call, the variants of a workload in alternation, `rounds` times; the JSON keeps every round and the median. The card name and power limit are read in the
same run.

    python tools/jvp_steps.py [--reps 20] [--rounds 5] [--out tools/jvp_steps_results.json]
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))

import torch  # noqa: E402
from torch import nn  # noqa: E402
from torch.func import jvp, vmap  # noqa: E402

import b200rnn  # noqa: E402

WORKLOADS = {
    "audio_gru256_b64": dict(cls=nn.GRU, I=256, H=256, L=2, bi=False, bf=True, B=64, T=120),
    "audio_gru256_b128": dict(cls=nn.GRU, I=256, H=256, L=2, bi=False, bf=True, B=128, T=120),
    "text_bilstm128": dict(cls=nn.LSTM, I=1024, H=128, L=2, bi=True, bf=False, B=64, T=30),
    "lstm512": dict(cls=nn.LSTM, I=512, H=512, L=1, bi=False, bf=False, B=16, T=120),
    "rnn_tanh256": dict(cls=nn.RNN, I=256, H=256, L=1, bi=False, bf=False, B=64, T=120),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"name": name, "power_limit": power}


def time_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "jvp_steps_results.json"))
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this tool measures on the GPU"
    dev = torch.device("cuda:0")
    result = {"card": card(), "reps": args.reps, "rounds": args.rounds, "workloads": {}}
    names = args.only.split(",") if args.only else list(WORKLOADS)
    for name in names:
        w = WORKLOADS[name]
        torch.manual_seed(0)
        stock = w["cls"](w["I"], w["H"], num_layers=w["L"], bidirectional=w["bi"], batch_first=w["bf"]).to(dev).eval()
        mine = b200rnn.from_torch(copy.deepcopy(stock)).to(dev).eval()
        shape = (w["B"], w["T"], w["I"]) if w["bf"] else (w["T"], w["B"], w["I"])
        x = torch.randn(shape, device=dev)
        v = torch.randn_like(x)
        f_mine = lambda x: mine(x)[0]  # noqa: E731
        f_stock = lambda x: stock(x)[0]  # noqa: E731

        def stock_nocudnn():
            with torch.backends.cudnn.flags(enabled=False):
                return jvp(f_stock, (x,), (v,))

        variants = {
            "b200rnn_forward": lambda: torch.no_grad()(f_mine)(x),
            "b200rnn_jvp": lambda: jvp(f_mine, (x,), (v,)),
        }
        row = {"shape": dict(w, cls=w["cls"].__name__)}
        stock_ok = {}
        # stock without and with cuDNN: a time, or what it raises
        for key, fn in (("stock_jvp_no_cudnn", stock_nocudnn), ("stock_jvp_cudnn", lambda: jvp(f_stock, (x,), (v,)))):
            try:
                stock_ok[key] = fn()[1]
                variants[key] = fn
            except Exception as e:  # noqa: BLE001
                row[key + "_error"] = f"{type(e).__name__}: {str(e).splitlines()[0][:300]}"
        _, ref = jvp(f_mine, (x,), (v,))
        for M in (8, 32):
            V = torch.randn(M, *x.shape, device=dev)
            variants[f"b200rnn_jacfwd_M{M}"] = (lambda V: lambda: vmap(lambda t: jvp(f_mine, (x,), (t,))[1])(V))(V)
            variants[f"b200rnn_jvp_loop_M{M}"] = (lambda V: lambda: [jvp(f_mine, (x,), (t,))[1] for t in V])(V)
            batched = vmap(lambda t: jvp(f_mine, (x,), (t,))[1])(V)
            looped = torch.stack([jvp(f_mine, (x,), (t,))[1] for t in V])
            row[f"jacfwd_M{M}_vs_loop_max_abs_diff"] = float((batched - looped).abs().max())
        for key, want in stock_ok.items():
            row[f"jvp_vs_{key}_rel_err"] = float((ref - want).abs().max() / want.abs().max())
        rounds = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                rounds[k].append(time_ms(fn, args.reps))
        row["ms_rounds"] = rounds
        row["ms_median"] = {k: statistics.median(r) for k, r in rounds.items()}
        result["workloads"][name] = row
        print(name, json.dumps(row["ms_median"]), flush=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
