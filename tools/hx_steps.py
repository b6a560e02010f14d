#!/usr/bin/env python
"""What an initial state costs: forward + backward with hx = None, with a given hx, and with dh_0 requested.

Two encoders of the fuse model, trainable, batch_first (as tools/varlen_steps.py):
  * audio GRU: B = 128, T = 120, I = H = 256, 2 layers;
  * text BiLSTM: B = 64, T = 30, I = 1024, H = 256, 2 layers.
Three cases each:
  * `none`: hx = None (the kernels start from zeros);
  * `hx`: a given hx that does not require grad (the backward pairs the first step with h_0 in dW_hh, no dh_0);
  * `hx_grad`: hx requires grad, so the backward also runs the last step's contraction for dh_0 / dc_0.
Per case: the whole forward + backward (CUDA events around `reps` iterations, profiling off), then the library's launches
alone (its profile hook: event pairs around each forward / backward recurrence launch and each GEMM).

    python tools/hx_steps.py [--reps 20] [--out FILE]     # B200RNN_LIB=... to time another build of the library
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

ENCODERS = {
    # name: (kind, B, T, I, H, bidirectional)
    "audio_gru": ("gru", 128, 120, 256, 256, False),
    "text_bilstm": ("lstm", 64, 30, 1024, 256, True),
}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "hx_steps.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    out = {"device": torch.cuda.get_device_name(dev), "nvidia_smi": gpu_info(), "library": _lib.LIB_PATH,
           "reps": args.reps, "encoders": {}}
    for name, (kind, B, T, I, H, bi) in ENCODERS.items():
        torch.manual_seed(0)
        cls = b200rnn.GRU if kind == "gru" else b200rnn.LSTM
        model = cls(I, H, num_layers=2, bidirectional=bi, batch_first=True).to(dev)
        D = 2 if bi else 1
        x = torch.randn(B, T, I, device=dev, requires_grad=True)
        states = [0.5 * torch.randn(2 * D, B, H, device=dev) for _ in range(1 if kind == "gru" else 2)]
        res = {"B": B, "T": T, "I": I, "H": H, "bidirectional": bi}
        for case in ("none", "hx", "hx_grad"):
            hx = None
            if case != "none":
                hs = [s.clone().requires_grad_(case == "hx_grad") for s in states]
                hx = hs[0] if kind == "gru" else tuple(hs)

            def step():
                y, st = model(x, hx)
                loss = y.square().sum()
                for s in (st if isinstance(st, tuple) else (st,)):
                    loss = loss + s.sum()
                loss.backward()

            for _ in range(3):
                step()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                step()
            e1.record()
            torch.cuda.synchronize()
            step_ms = e0.elapsed_time(e1) / args.reps
            _lib.profile(True)
            for _ in range(args.reps):
                step()
            torch.cuda.synchronize()
            fwd_ms, fwd_n = _lib.profile_read(_lib.PROF_REC_FWD)
            bwd_ms, bwd_n = _lib.profile_read(_lib.PROF_REC_BWD)
            gemm_ms, gemm_n = _lib.profile_read(_lib.PROF_GEMM)
            _lib.profile(False)
            res[case] = {"fwd_bwd_ms": step_ms,
                         "rec_fwd_ms_per_launch": fwd_ms / max(fwd_n, 1), "rec_fwd_launches": fwd_n,
                         "rec_bwd_ms_per_launch": bwd_ms / max(bwd_n, 1), "rec_bwd_launches": bwd_n,
                         "gemm_ms_per_step": gemm_ms / args.reps, "gemm_launches_per_step": gemm_n / args.reps}
        out["encoders"][name] = res
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
