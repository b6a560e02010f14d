"""Eager against ``torch.compile`` for the forward + backward of the BASELINE c2 audio model (``AudioBiLSTM``,
B = 64, T = 120, 256-d, H = 256) and the c3 text model (``TextBiLSTM``, B = 64, T = 30, 1024-d, H = 256), in train
mode with dropout.

Compiled, the RNN runs through the ``b200rnn::`` custom ops and the shell through inductor; the shell fusions of the
eager models (``forward_ln_sum``'s fused LayerNorm / time sum, the attention-pooling kernels) are not taken. Each
round times ``--iters`` calls of each variant with CUDA events, the two alternated; the result is the median over
``--rounds`` rounds, in ms per call. Writes tools/compile_steps_results.json unless ``--out`` says otherwise.

    python tools/compile_steps.py [--rounds 7] [--iters 20] [--out PATH]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))

import torch  # noqa: E402

import b200rnn  # noqa: E402


def _model(kind, dev):
    torch.manual_seed(0)
    if kind == "c2":
        cfg = dict(num_classes=2, dropout=0.5, rnn_layers=2, embedding_size=256, hidden_dims=256)
        return b200rnn.AudioBiLSTM(cfg).to(dev).train(), torch.randn(64, 120, 256, device=dev, requires_grad=True)
    cfg = dict(num_classes=2, dropout=0.5, rnn_layers=2, embedding_size=1024, hidden_dims=256, bidirectional=True)
    return b200rnn.TextBiLSTM(cfg).to(dev).train(), torch.randn(64, 30, 1024, device=dev, requires_grad=True)


def _time(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def measure(kind, rounds, iters, dev):
    model, x = _model(kind, dev)
    labels = torch.randint(0, 2, (64,), device=dev)
    crit = torch.nn.CrossEntropyLoss()
    compiled = torch.compile(model)

    def step(m):
        def run():
            crit(m(x), labels).backward()
        return run

    eager_step, compiled_step = step(model), step(compiled)
    for _ in range(3):            # compile, warm the allocator and both paths
        eager_step()
        compiled_step()
    torch.cuda.synchronize()
    eager, comp = [], []
    for _ in range(rounds):
        eager.append(_time(eager_step, iters))
        comp.append(_time(compiled_step, iters))
    med_e, med_c = statistics.median(eager), statistics.median(comp)
    return {"eager_ms": round(med_e, 4), "compiled_ms": round(med_c, 4), "compiled_over_eager": round(med_c / med_e, 4),
            "eager_rounds_ms": [round(v, 4) for v in eager], "compiled_rounds_ms": [round(v, 4) for v in comp]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                  "compile_steps_results.json"))
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(dev), "torch": torch.__version__,
           "what": "forward + backward of the model in train mode, ms per call, median of alternated rounds",
           "rounds": args.rounds, "iters_per_round": args.iters,
           "c2_audio_B64_T120_H256": measure("c2", args.rounds, args.iters, dev),
           "c3_text_B64_T30_H256": measure("c3", args.rounds, args.iters, dev)}
    print(json.dumps(res, indent=1))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
