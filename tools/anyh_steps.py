#!/usr/bin/env python
"""What the runtime-sized recurrence (csrc/rnn_anyh.cu) costs per layer launch, against stock cuDNN.

One unidirectional layer, time-major, T = 120, I = 64, for H in {64, 192, 384, 512, 1024}, GRU and LSTM, B in
{16, 64, 128}:
  * `ours`: b200rnn.GRU / LSTM: the forward and backward recurrence launches alone (the library's profile hook: event
    pairs around each launch), the whole forward + backward of the module (CUDA events around `reps` calls), and the
    config the library chose (B200RNN_DEBUG line, read from a subprocess: cluster width C, batch rows BS, weight tier);
  * `cudnn_fp32` / `cudnn_tf32`: stock torch.nn.GRU / LSTM(...).cuda() with cuDNN's RNN math in IEEE fp32
    (torch.backends.cudnn.rnn.fp32_precision = "ieee") and in TF32 ("tf32", torch's default): forward alone and
    forward + backward (CUDA events).
They are timed in alternation, `rounds` times, after a warm-up; the JSON keeps every round. The card name, its power
limit and clocks are read in the same run.

    python tools/anyh_steps.py [--reps 10] [--rounds 3] [--out tools/anyh_steps_results.json]
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

HS = (64, 192, 384, 512, 1024)
BS = (16, 64, 128)
T, I = 120, 64


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
    s = out[1] if isinstance(out[1], tuple) else (out[1],)
    return out[0].square().sum() + sum(v.sum() for v in s)


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
    return {"rec_fwd_us_per_launch": 1e3 * fwd_ms / max(fwd_n, 1), "rec_bwd_us_per_launch": 1e3 * bwd_ms / max(bwd_n, 1),
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


_CFG = r"""
import sys, torch, b200rnn
T, I = int(sys.argv[1]), int(sys.argv[2])
for spec in sys.argv[3:]:
    kind, H, B = spec.split(":")
    print("SHAPE", spec, file=sys.stderr, flush=True)
    m = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(I, int(H)).cuda()
    x = torch.randn(T, int(B), I, device="cuda", requires_grad=True)
    m(x)[0].sum().backward()
    torch.cuda.synchronize()
"""


def chosen_configs(specs):
    """{"kind:H:B": [the B200RNN_DEBUG config lines of one forward + backward]}, from one subprocess"""
    env = dict(os.environ, B200RNN_DEBUG="1")
    r = subprocess.run([sys.executable, "-c", _CFG, str(T), str(I), *specs], capture_output=True, text=True, env=env,
                       cwd=os.path.join(ROOT, "icassp2022-depression_b200"), timeout=600)
    out, cur = {}, None
    for ln in r.stderr.splitlines():
        if ln.startswith("SHAPE "):
            cur = ln.split()[1]
            out[cur] = []
        elif cur and re.search(r"(fwd|bwd) (anyh )?cfg", ln):
            out[cur].append(ln)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "anyh_steps.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    out = {"device": torch.cuda.get_device_name(dev), "nvidia_smi": gpu_info(),
           "library": os.path.relpath(_lib.LIB_PATH, ROOT), "T": T, "I": I, "bidirectional": False, "num_layers": 1,
           "reps": args.reps, "cudnn": "torch.nn.GRU/LSTM(...).cuda(); cudnn_fp32: rnn.fp32_precision='ieee', "
           "cudnn_tf32: 'tf32'", "shapes": []}
    configs = chosen_configs([f"{k}:{H}:{B}" for k in ("gru", "lstm") for H in HS for B in BS])
    for kind in ("gru", "lstm"):
        stock = b200rnn.modules._TORCH_GRU if kind == "gru" else b200rnn.modules._TORCH_LSTM
        for H in HS:
            for B in BS:
                torch.manual_seed(0)
                x = torch.randn(T, B, I, device=dev, requires_grad=True)
                mine = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(I, H).to(dev)
                ref = stock(I, H).to(dev)
                res = {"kind": kind, "H": H, "B": B, "config": configs.get(f"{kind}:{H}:{B}"),
                       "rounds": {"ours": [], "cudnn_fp32": [], "cudnn_tf32": []}}
                for _ in range(args.rounds):
                    res["rounds"]["ours"].append(ours(mine, x, args.reps))
                    res["rounds"]["cudnn_fp32"].append(cudnn(ref, x, args.reps, "ieee"))
                    res["rounds"]["cudnn_tf32"].append(cudnn(ref, x, args.reps, "tf32"))
                out["shapes"].append(res)
                print(json.dumps(res), flush=True)
    text = json.dumps(out, indent=1)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
