#!/usr/bin/env python
"""Where does the audio chain of the fuse step wait? (one GPU, CUDA-graph replays under torch.profiler)

Captures bench.py's two-stream fuse step (`FusedFuseStep`, B = 128, bench.py's synthetic inputs) and, for reference,
the audio branch alone, as CUDA graphs; after a warm-up it profiles `--replays` replays of each with CUDA activities.
Every kernel's stream, grid, start and end (µs, relative to its replay's first kernel) go to
`<out>/step_timeline.json`; the raw chrome traces go beside it.

The audio chain is the stream that runs the GRU recurrence (`rec_fwd_tc_kernel`, or `rec_fwd_h16_kernel` in the
no-grad fused forward); every other kernel of the step is the text branch or the head. For each audio kernel it
prints, as medians over the replays:
  * `gap`: its start minus the end of its predecessor on the audio stream (negative for a recurrence that starts
    beside its streamed GEMM); for a recurrence also `after_gemm_start`;
  * its duration, beside its duration when the audio branch runs alone.
and the end of the text branch (with the text half of the head) relative to the end of the audio chain (negative: the
text branch ends first). The head launch after the join (the step's last kernel) is counted in neither: it is
listed on its own, with the join gap (its start minus the end of everything before it) and the time from the audio
chain's end to the step's end. The text-branch kernels (every kernel
off the audio stream before the join) are listed too, in start order: name, grid, median start and duration, so that
what runs beside rec0's end and rec1's start can be read off, each beside its duration when the text branch runs
alone.

    python tools/step_timeline.py [--replays 20] [--out DIR]      # default DIR: step_timeline/ in the temp directory
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))
os.environ.setdefault("OMP_NUM_THREADS", "1")

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import b200rnn  # noqa: E402
import bench  # noqa: E402

# the GRU-256 forward recurrence: 3xTF32 tensor cores, or fp16 pairs in the no-grad fused forward
REC = ("rec_fwd_tc_kernel", "rec_fwd_h16_kernel")
# the head launch after the join: the whole head, or only the loss / dW / Adam of the split classification head
AFTER_JOIN = ("fuse_head_kernel", "fuse_loss_kernel")


def _card():
    """Name, power limit and max SM clock, read in the same run as the timeline."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def _capture(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn(0)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graphs, pool = [], None
    for i in range(bench.N_ROTATE):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, pool=pool):
            fn(i)
        pool = g.pool()
        graphs.append(g)
    return graphs


def _kernels(run, replays, warmup, trace_path):
    """Per replay, the list of kernels {name, stream, grid, start, end} sorted by start (µs from the first start).
    ``run(i)`` enqueues step i."""
    for i in range(warmup):
        run(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(replays):
            run(i)
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace_path)
    return _parse(trace_path, replays)


def _parse(trace_path, replays):
    with open(trace_path) as f:
        ev = json.load(f)
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    ks = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    if not ks or len(ks) % replays:
        raise RuntimeError(f"{len(ks)} kernels in the trace of {replays} replays")
    n = len(ks) // replays
    out = []
    for r in range(replays):  # graph launches are stream-ordered: replay r+1 starts after all of replay r has ended
        chunk = ks[r * n:(r + 1) * n]
        t0 = chunk[0]["ts"]
        out.append([{"name": re.search(r"(\w+)\s*[<(]", e["name"]).group(1), "stream": e["args"].get("stream"),
                     "grid": e["args"].get("grid"), "start": e["ts"] - t0, "end": e["ts"] + e["dur"] - t0}
                    for e in chunk])
    return out


def _median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2] if len(xs) % 2 else 0.5 * (xs[len(xs) // 2 - 1] + xs[len(xs) // 2])


def _split(replay):
    """(audio chain, text branch, after the join): the kernels on the recurrence's stream; the others; the step's last
    launch, the head kernel that runs once both branches have ended. A replayed graph may report that kernel on either
    branch's stream, so it is told apart by its place, not its stream."""
    streams = {k["stream"] for k in replay if k["name"] in REC}
    if len(streams) != 1:
        raise RuntimeError(f"the GRU recurrences ran on streams {sorted(streams)}; expected one audio stream")
    s = streams.pop()
    before, post = (replay[:-1], replay[-1:]) if replay[-1]["name"] in AFTER_JOIN else (replay, [])
    return [k for k in before if k["stream"] == s], [k for k in before if k["stream"] != s], post


def _audio_chain(replay):
    """(audio chain, text branch): the kernels on the recurrence's stream, and the others; the kernels after the join
    belong to neither."""
    audio, other, _ = _split(replay)
    return audio, other


def _post_join(replays):
    """The kernels after the join (name, grid, median start and duration, µs), the median join gap (first post-join
    start minus the end of every kernel before it) and the median time from the audio chain's end to the step's end."""
    parts = [_split(r) for r in replays]
    names = [k["name"] for k in parts[0][2]]
    if any([k["name"] for k in p[2]] != names for p in parts):
        raise RuntimeError("the kernels after the join differ between replays")
    rows = [{"kernel": n, "grid": parts[0][2][i]["grid"],
             "start_us": round(_median([p[2][i]["start"] for p in parts]), 1),
             "dur_us": round(_median([p[2][i]["end"] - p[2][i]["start"] for p in parts]), 1)}
            for i, n in enumerate(names)]
    gap = _median([p[2][0]["start"] - max(k["end"] for k in p[0] + p[1]) for p in parts]) if names else 0.0
    tail = _median([max(k["end"] for k in r) - max(k["end"] for k in p[0]) for r, p in zip(replays, parts)])
    return rows, round(gap, 1), round(tail, 1)


def _chain_rows(replays):
    """Per position of the audio chain: name, median gap to its predecessor, median duration (µs)."""
    chains = [_audio_chain(r) for r in replays]
    n = len(chains[0][0])
    if any(len(a) != n for a, _ in chains):
        raise RuntimeError("the audio chain has a different number of kernels in different replays")
    rows = []
    for i in range(n):
        ks = [a[i] for a, _ in chains]
        row = {"kernel": ks[0]["name"], "grid": ks[0]["grid"],
               "start_us": round(_median([k["start"] for k in ks]), 1),
               "dur_us": round(_median([k["end"] - k["start"] for k in ks]), 1)}
        if i > 0:
            row["gap_us"] = round(_median([a[i]["start"] - a[i - 1]["end"] for a, _ in chains]), 1)
            if ks[0]["name"] in REC:
                row["after_gemm_start_us"] = round(_median([a[i]["start"] - a[i - 1]["start"] for a, _ in chains]), 1)
        rows.append(row)
    text_end = [max((k["end"] for k in o), default=0.0) - a[-1]["end"] for a, o in chains]
    step = [max(k["end"] for k in r) for r in replays]
    return rows, _median(text_end), _median(step), _text_rows(chains)


def _text_rows(chains):
    """Per position of the text branch (kernels off the audio stream, in start order): name, grid, median start and
    duration (µs). Empty when the replays disagree on its kernels."""
    texts = [o for _, o in chains]
    n = len(texts[0])
    if any(len(o) != n or [k["name"] for k in o] != [k["name"] for k in texts[0]] for o in texts):
        return []
    return [{"kernel": texts[0][i]["name"], "grid": texts[0][i]["grid"],
             "start_us": round(_median([o[i]["start"] for o in texts]), 1),
             "dur_us": round(_median([o[i]["end"] - o[i]["start"] for o in texts]), 1)} for i in range(n)]


def _alone_rows(replays):
    """Per position of a replay that runs one branch alone: name, grid, median duration (µs)"""
    n = len(replays[0])
    if any(len(r) != n for r in replays):
        raise RuntimeError("the branch has a different number of kernels in different replays")
    return [{"kernel": replays[0][i]["name"], "grid": replays[0][i]["grid"],
             "dur_us": round(_median([r[i]["end"] - r[i]["start"] for r in replays]), 1)} for i in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "step_timeline"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("step_timeline.py needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.set_num_threads(1)
    torch.manual_seed(0)
    card = _card()
    model = b200rnn.fusion_net(**bench.FUSE_ARGS).to(dev)
    for p in model.parameters():
        p.requires_grad = False
    model.fc_final[0].weight.requires_grad = True
    model.train()
    host = [bench._synthetic(bench.B_PER_GPU, 1234 + i) for i in range(bench.N_ROTATE)]
    dev_in = [(a.to(dev), t.to(dev), y.to(dev)) for a, t, y in host]
    fused = b200rnn.FusedFuseStep(model, lr=bench.LR, exchange="none", concurrent_branches=True)

    def step(i):
        fused(b200rnn.FuseBatch(dev_in[i % bench.N_ROTATE][0], dev_in[i % bench.N_ROTATE][1]),
              dev_in[i % bench.N_ROTATE][2])

    def audio_branch(i):
        with torch.no_grad():
            fused._audio_branch(b200rnn.FuseBatch(dev_in[i % bench.N_ROTATE][0], dev_in[i % bench.N_ROTATE][1]))

    def text_branch(i):
        with torch.no_grad():
            fused._text_branch(b200rnn.FuseBatch(dev_in[i % bench.N_ROTATE][0], dev_in[i % bench.N_ROTATE][1]))

    whole, audio, text = _capture(step), _capture(audio_branch), _capture(text_branch)
    mode = "graph"
    runs = {"whole_step": _kernels(lambda i: whole[i % len(whole)].replay(), args.replays, args.warmup,
                                   os.path.join(args.out, "trace_whole.json")),
            "audio_alone": _kernels(lambda i: audio[i % len(audio)].replay(), args.replays, args.warmup,
                                    os.path.join(args.out, "trace_audio.json")),
            "text_alone": _kernels(lambda i: text[i % len(text)].replay(), args.replays, args.warmup,
                                   os.path.join(args.out, "trace_text.json"))}
    if len({k["stream"] for k in runs["whole_step"][0]}) < 2:
        # the profiler put every kernel of the graph on the launching stream: fall back to eager steps, whose
        # kernels carry the stream they were enqueued on
        mode = "eager"
        runs = {"whole_step": _kernels(step, args.replays, args.warmup, os.path.join(args.out, "trace_whole.json")),
                "audio_alone": _kernels(audio_branch, args.replays, args.warmup,
                                        os.path.join(args.out, "trace_audio.json")),
                "text_alone": _kernels(text_branch, args.replays, args.warmup, os.path.join(args.out, "trace_text.json"))}
    rows, text_end, step, text_rows = _chain_rows(runs["whole_step"])
    alone, _, audio_step, _ = _chain_rows(runs["audio_alone"])
    if len(rows) < len(alone):
        raise RuntimeError("the audio chain differs between the whole step and the audio branch alone")
    for r, a in zip(rows, alone):  # kernels past the audio branch alone (the head's audio stage) have no alone value
        if r["kernel"] != a["kernel"]:
            raise RuntimeError("the audio chain differs between the whole step and the audio branch alone")
        r["dur_alone_us"] = a["dur_us"]
        if "gap_us" in a:
            r["gap_alone_us"] = a["gap_us"]
    text_alone = _alone_rows(runs["text_alone"])  # the text half of the head is not part of the text branch alone
    if [r["kernel"] for r in text_rows[:len(text_alone)]] == [a["kernel"] for a in text_alone]:
        for r, a in zip(text_rows, text_alone):
            r["dur_alone_us"] = a["dur_us"]
    post, join_gap, tail = _post_join(runs["whole_step"])
    summary = {"card": card, "mode": mode, "replays": args.replays, "audio_chain": rows, "text_branch": text_rows,
               "text_end_minus_audio_end_us": round(text_end, 1), "post_join": post, "join_gap_us": join_gap,
               "audio_end_to_step_end_us": tail, "whole_step_us": round(step, 1),
               "audio_alone_us": round(audio_step, 1)}
    with open(os.path.join(args.out, "step_timeline.json"), "w") as f:
        json.dump({"summary": summary, "kernels": runs}, f, indent=1)
    print(f"card: {card}; {mode} steps")
    print(f"{'audio kernel':<22}{'grid':>16}{'start':>9}{'gap':>9}{'gap alone':>11}{'dur':>9}{'dur alone':>11}"
          f"{'after GEMM start':>18}   (µs, median of {args.replays} replays)")
    for r in rows:
        print(f"{r['kernel'][:21]:<22}{str(r['grid']):>16}{r['start_us']:>9}{r.get('gap_us', ''):>9}"
              f"{r.get('gap_alone_us', ''):>11}{r['dur_us']:>9}{r.get('dur_alone_us', ''):>11}"
              f"{r.get('after_gemm_start_us', ''):>18}")
    print(f"{'text kernel':<22}{'grid':>16}{'start':>9}{'dur':>9}{'end':>9}{'dur alone':>11}")
    for r in text_rows:
        print(f"{r['kernel'][:21]:<22}{str(r['grid']):>16}{r['start_us']:>9}{r['dur_us']:>9}"
              f"{round(r['start_us'] + r['dur_us'], 1):>9}{r.get('dur_alone_us', ''):>11}")
    if not text_rows:
        print("text alone: " + ", ".join(f"{a['kernel']} {a['grid']} {a['dur_us']}" for a in text_alone))
    print(f"{'after the join':<22}{'grid':>16}{'start':>9}{'dur':>9}")
    for r in post:
        print(f"{r['kernel'][:21]:<22}{str(r['grid']):>16}{r['start_us']:>9}{r['dur_us']:>9}")
    print(f"join gap {join_gap} µs; audio chain end to step end {tail} µs")
    print(f"text branch ends {text_end:+.1f} µs after the audio chain; step (first to last kernel) {step:.1f} µs, "
          f"audio branch alone {audio_step:.1f} µs")
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
