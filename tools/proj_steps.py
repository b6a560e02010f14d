#!/usr/bin/env python
"""What a projection (LSTMP, proj_size) costs, per layer launch, at the text branch's shapes.

One bidirectional layer, batch_first, T = 30, I = 1024, B = 64 and 128, for each supported (H, P):
  * `proj`: b200rnn.LSTM(proj_size=P): the library's forward / backward recurrence launches alone (its profile hook:
    event pairs around each launch) and the whole forward + backward of the module (CUDA events around `reps` calls);
  * `plain`: b200rnn.LSTM at the same H without a projection, the same numbers;
  * `cudnn`: stock torch.nn.LSTM(proj_size=P).cuda(): forward alone and forward + backward (CUDA events).
The three are timed in alternation, `rounds` times, after a warm-up; the JSON keeps every round. The card name and its
power limit are read in the same run.

    python tools/proj_steps.py [--reps 20] [--rounds 3] [--out tools/proj_steps_results.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))

import torch  # noqa: E402

import b200rnn  # noqa: E402
from b200rnn import _lib  # noqa: E402

SIZES = [(128, 32), (128, 64), (256, 64), (256, 128)]
T, I = 30, 1024


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


def ours(model, x, reps):
    def step():
        y, (h, c) = model(x)
        (y.square().sum() + h.sum() + c.sum()).backward()

    for _ in range(3):
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
    return {"rec_fwd_us_per_launch": 1e3 * fwd_ms / max(fwd_n, 1), "rec_bwd_us_per_launch": 1e3 * bwd_ms / max(bwd_n, 1),
            "fwd_bwd_ms": step_ms}


def cudnn(model, x, reps):
    def fwd():
        with torch.no_grad():
            model(x)

    def step():
        y, (h, c) = model(x)
        (y.square().sum() + h.sum() + c.sum()).backward()

    for _ in range(3):
        fwd()
        step()
    torch.cuda.synchronize()
    return {"fwd_ms": timed(fwd, reps), "fwd_bwd_ms": timed(step, reps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "proj_steps.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    out = {"device": torch.cuda.get_device_name(dev), "nvidia_smi": gpu_info(),
           "library": os.path.relpath(_lib.LIB_PATH, ROOT),
           "T": T, "I": I, "bidirectional": True, "num_layers": 1, "reps": args.reps, "shapes": []}
    for B in (64, 128):
        for H, P in SIZES:
            torch.manual_seed(0)
            x = torch.randn(B, T, I, device=dev, requires_grad=True)
            models = {
                "proj": b200rnn.LSTM(I, H, bidirectional=True, batch_first=True, proj_size=P).to(dev),
                "plain": b200rnn.LSTM(I, H, bidirectional=True, batch_first=True).to(dev),
                "cudnn": b200rnn.modules._TORCH_LSTM(I, H, bidirectional=True, batch_first=True, proj_size=P).to(dev),
            }
            res = {"B": B, "H": H, "P": P, "rounds": {k: [] for k in models}}
            for _ in range(args.rounds):
                for k, m in models.items():
                    res["rounds"][k].append((cudnn if k == "cudnn" else ours)(m, x, args.reps))
            out["shapes"].append(res)
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
