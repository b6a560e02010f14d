"""Time the 16-bit modules against the fp32 modules and stock cuDNN in the same dtype.

Per shape and per variant (ours in f16 / bf16, ours in fp32, cuDNN in f16 / bf16): the module forward and the
forward + backward (CUDA events around whole calls, ms per call), and for our modules the device time per recurrence
launch and per GEMM launch, forward and backward (the library's own event pairs, b200rnn_profile). Rounds alternate
the variants so that clock drift and neighbours on the machine hit all of them alike. The card, its power limit and
max SM clock are read in the same run and stored beside the numbers.

    python tools/h16_module_steps.py --out tools/h16_module_steps_results.json [--rounds 3] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))
import b200rnn  # noqa: E402
from b200rnn import _lib  # noqa: E402

# the reference sizes, then the sizes whose W_hh moves on chip in 16 bits (forward bound: GRU 752, LSTM 640)
SHAPES = [
    dict(kind="gru", I=256, H=256, L=2, bi=False, B=128, T=120),
    dict(kind="lstm", I=1024, H=128, L=2, bi=True, B=128, T=30),
    dict(kind="lstm", I=1024, H=256, L=2, bi=True, B=128, T=30),
    dict(kind="lstm", I=256, H=512, L=1, bi=False, B=16, T=120),
    dict(kind="lstm", I=256, H=512, L=1, bi=False, B=128, T=120),
    dict(kind="gru", I=256, H=640, L=1, bi=False, B=16, T=120),
    dict(kind="gru", I=256, H=720, L=1, bi=False, B=16, T=120),
    dict(kind="gru", I=256, H=720, L=1, bi=False, B=128, T=120),
]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def build(s, variant):
    cls = {"gru": (b200rnn.GRU, torch.nn.GRU), "lstm": (b200rnn.LSTM, torch.nn.LSTM)}[s["kind"]]
    dt = {"ours_f16": torch.float16, "ours_bf16": torch.bfloat16, "ours_f32": torch.float32,
          "cudnn_f16": torch.float16, "cudnn_bf16": torch.bfloat16}[variant]
    mod = (cls[1] if variant.startswith("cudnn") else cls[0])(s["I"], s["H"], num_layers=s["L"],
                                                              bidirectional=s["bi"], dtype=dt).cuda()
    x = torch.randn(s["T"], s["B"], s["I"], device="cuda").to(dt).requires_grad_(True)
    return mod, x


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def per_launch(mod, x, iters):
    """device ms per launch of our recurrence (fwd, bwd) and GEMMs over one forward + backward"""
    _lib.profile(True)
    for _ in range(iters):
        mod(x)[0].float().sum().backward()
    torch.cuda.synchronize()
    out = {}
    for name, kind in (("rec_fwd", _lib.PROF_REC_FWD), ("rec_bwd", _lib.PROF_REC_BWD), ("gemm", _lib.PROF_GEMM),
                       ("other", _lib.PROF_MISC)):
        ms, n = _lib.profile_read(kind)
        out[name] = {"ms_per_launch": ms / n if n else None, "launches_per_step": n / iters}
    _lib.profile(False)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    variants = ["ours_f16", "ours_bf16", "ours_f32", "cudnn_f16", "cudnn_bf16"]
    res = {"card": card(), "rounds": args.rounds, "iters": args.iters, "shapes": []}
    for s in SHAPES:
        built = {v: build(s, v) for v in variants}
        rec = {v: {"fwd_ms": [], "fwd_bwd_ms": []} for v in variants}
        for _ in range(args.rounds):
            for v in variants:
                mod, x = built[v]
                with torch.no_grad():
                    rec[v]["fwd_ms"].append(timed(lambda: mod(x), args.iters))
                rec[v]["fwd_bwd_ms"].append(timed(lambda: mod(x)[0].float().sum().backward(), args.iters))
        for v in variants:
            if v.startswith("ours"):
                rec[v]["launches"] = per_launch(*built[v], args.iters)
        res["shapes"].append({"shape": s, "results": rec})
        print(json.dumps({"shape": s, **{v: [min(rec[v]["fwd_ms"]), min(rec[v]["fwd_bwd_ms"])] for v in variants}}),
              flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
