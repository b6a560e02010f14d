#!/usr/bin/env python
"""Forward + backward time of ragged batches: what skipping the padded tail of each cluster saves.

Two encoders of the fuse model, trainable, batch_first:
  * audio GRU: B = 128, T = 120, I = H = 256, 2 layers;
  * text BiLSTM: B = 64, T = 30, I = 1024, H = 256, 2 layers.
Three inputs each:
  * `skewed`: packed, DAIC-like lengths (one participant answers at length, most briefly: log-normal around T / 4,
    one row at T, rows in random order);
  * `full`: packed, every length T (the slot order is the identity, every cluster runs T steps);
  * `dense`: the padded tensor, no lengths.
Per case: the whole forward + backward (CUDA events around `reps` iterations, profiling off), then the recurrence
launches alone (the library's profile hook: event pairs around each forward / backward recurrence launch).
`slice_steps_share` is what the recurrence time should scale with: the sum over batch slices of BS rows of the slice's
longest length, over nslices * T, for each BS the configs use.

    python tools/varlen_steps.py [--reps 20]      # B200RNN_LIB=... to time another build of the library
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))

import torch  # noqa: E402
from torch.nn.utils.rnn import pack_padded_sequence  # noqa: E402

import b200rnn  # noqa: E402
from b200rnn import _lib  # noqa: E402

ENCODERS = {
    # name: (kind, B, T, I, H, bidirectional)
    "audio_gru": ("gru", 128, 120, 256, 256, False),
    "text_bilstm": ("lstm", 64, 30, 1024, 256, True),
}


def daic_like_lengths(B, T, gen):
    """log-normal lengths with median T / 4, clipped to [1, T], one row at T, in random row order"""
    lens = torch.exp(math.log(T / 4) + 0.6 * torch.randn(B, generator=gen)).round().clamp(1, T).long()
    lens[int(torch.randint(0, B, (1,), generator=gen))] = T
    return lens


def slice_steps_share(lens, T, BS):
    s = torch.sort(lens, descending=True, stable=True).values
    heads = s[::BS]
    return heads.sum().item() / (len(heads) * T)


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
    args = ap.parse_args()
    assert torch.cuda.is_available(), "varlen_steps.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    out = {"device": torch.cuda.get_device_name(dev), "nvidia_smi": gpu_info(), "library": _lib.LIB_PATH,
           "reps": args.reps, "encoders": {}}
    gen = torch.Generator().manual_seed(0)
    for name, (kind, B, T, I, H, bi) in ENCODERS.items():
        torch.manual_seed(0)
        cls = b200rnn.GRU if kind == "gru" else b200rnn.LSTM
        model = cls(I, H, num_layers=2, bidirectional=bi, batch_first=True).to(dev)
        x = torch.randn(B, T, I, device=dev, requires_grad=True)
        skewed = daic_like_lengths(B, T, gen)
        res = {"B": B, "T": T, "I": I, "H": H, "bidirectional": bi,
               "skewed_lengths": {"mean": skewed.float().mean().item(), "max": int(skewed.max()),
                                  "slice_steps_share": {bs: slice_steps_share(skewed, T, bs) for bs in (2, 4, 8)}}}
        cases = {"skewed": skewed, "full": torch.full((B,), T), "dense": None}
        for case, lens in cases.items():
            def step():
                inp = x if lens is None else pack_padded_sequence(x, lens, batch_first=True, enforce_sorted=False)
                y = model(inp)[0]
                (y.data if lens is not None else y).square().sum().backward()

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
            _lib.profile(False)
            res[case] = {"fwd_bwd_ms": step_ms,
                         "rec_fwd_ms_per_launch": fwd_ms / max(fwd_n, 1), "rec_fwd_launches": fwd_n,
                         "rec_bwd_ms_per_launch": bwd_ms / max(bwd_n, 1), "rec_bwd_launches": bwd_n}
        out["encoders"][name] = res
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
