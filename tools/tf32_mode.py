"""Single-pass TF32 mode against the default 3xTF32, both alternated in one process on the current GPU.

For each mode (torch.backends.cuda.matmul.fp32_precision "ieee" -> 3xTF32, "tf32" -> single-pass TF32):
  * the two encoder branches of the fuse step (FusedFuseStep.features, B = 128, audio [128,120,256], text [128,30,1024],
    as bench.py builds them) as one CUDA-graph replay, ms;
  * the audio GRU-256 forward alone (B = 128, T = 120, 2 layers: streamed GEMM + tc8) and a c2-shape GRU training
    forward + backward (B = 64, T = 120: GEMMs + bs4), ms;
  * the error of the GRU output and of every gradient against float64 (oracle/rnn_numpy.py);
and, as a yardstick, stock torch.nn.GRU on CUDA (cuDNN at its default TF32 setting) on the same inputs.

    python tools/tf32_mode.py [--rounds 5] [--out tools/tf32_mode_results.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "icassp2022-depression_b200")]

import b200rnn  # noqa: E402
from oracle.rnn_numpy import NumpyRNN  # noqa: E402

DEV = "cuda:0"


def set_mode(mode):
    torch.backends.cuda.matmul.fp32_precision = mode


def gpu_info():
    q = "name,power.limit,clocks.max.sm,driver_version"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock, driver = [s.strip() for s in out.split(",")]
    except Exception as e:  # noqa: BLE001
        name, power, clock, driver = torch.cuda.get_device_name(0), f"unknown ({e})", "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock, "driver": driver, "torch": torch.__version__}


def time_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def capture(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def errors(kind, ref, mine, x, lengths=None):
    """max |y - y64|, max relative |dW - dW64| over all weights, |dx - dx64| relative."""
    w64 = [p.detach().double().numpy() for p in ref.parameters()]
    orc = NumpyRNN(kind, w64, ref.num_layers, ref.bidirectional)
    y64 = orc.forward(x.double().numpy().transpose(1, 0, 2))[0].transpose(1, 0, 2)
    dy = torch.randn(y64.shape, generator=torch.Generator().manual_seed(1))
    dx64, dp64 = orc.backward(dy.double().numpy().transpose(1, 0, 2))
    xm = x.to(DEV).requires_grad_(True)
    for p in mine.parameters():
        p.grad = None
    y = mine(xm)[0]
    (y * dy.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    err_y = float(np.abs(y.detach().cpu().double().numpy() - y64).max())
    err_dx = float(np.abs(xm.grad.cpu().double().numpy() - dx64.transpose(1, 0, 2)).max() / np.abs(dx64).max())
    err_w = max(float(np.abs(p.grad.cpu().double().numpy() - g).max() / np.abs(g).max())
                for p, g in zip(mine.parameters(), dp64))
    return {"y_abs": err_y, "dx_rel": err_dx, "dW_rel": err_w}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "tf32_mode_results.json"))
    args = ap.parse_args()
    torch.manual_seed(0)
    res = {"device": gpu_info(), "rounds": args.rounds, "iters": args.iters}

    # fuse step encoders, as bench.py builds them (eval: no dropout draws)
    m = b200rnn.fusion_net(1024, 128, 2, 0.3, 2, 256, 256).to(DEV).eval()
    for p in m.parameters():
        p.requires_grad = False
    m.fc_final[0].weight.requires_grad = True
    step = b200rnn.FusedFuseStep(m, exchange="none")
    batch = b200rnn.FuseBatch(torch.randn(128, 120, 256, device=DEV), torch.randn(128, 30, 1024, device=DEV))
    # audio GRU alone and the c2 training shape
    ref_a = torch.nn.GRU(256, 256, num_layers=2, batch_first=True)
    gru_a = b200rnn.from_torch(ref_a).to(DEV).eval()
    xa = torch.randn(128, 120, 256, device=DEV)
    gru_c2 = b200rnn.from_torch(ref_a).to(DEV).train()
    xc2 = torch.randn(64, 120, 256, device=DEV, requires_grad=True)
    dyc2 = torch.randn(64, 120, 256, device=DEV)

    def c2_step():
        y = gru_c2(xc2)[0]
        torch.autograd.backward(y, dyc2)

    graphs = {}
    for mode in ("ieee", "tf32"):
        set_mode(mode)
        with torch.no_grad():
            graphs[mode] = (capture(lambda: step.features(batch)), capture(lambda: gru_a(xa)))

    timings = {mode: {"fuse_features_graph_ms": [], "audio_gru_fwd_graph_ms": [], "c2_gru_fwd_bwd_ms": []}
               for mode in graphs}
    for _ in range(args.rounds):
        for mode in ("ieee", "tf32"):
            set_mode(mode)
            g_fuse, g_gru = graphs[mode]
            t = timings[mode]
            t["fuse_features_graph_ms"].append(time_ms(g_fuse.replay, args.iters))
            with torch.no_grad():
                t["audio_gru_fwd_graph_ms"].append(time_ms(g_gru.replay, args.iters))
            t["c2_gru_fwd_bwd_ms"].append(time_ms(c2_step, max(1, args.iters // 5)))
    res["timings_ms"] = {mode: {k: {"median": float(np.median(v)), "all": v} for k, v in t.items()}
                         for mode, t in timings.items()}

    # accuracy against float64 on one audio-shape batch (T shortened to keep the float64 oracle quick)
    x = torch.randn(128, 40, 256)
    acc = {}
    for mode in ("ieee", "tf32"):
        set_mode(mode)
        acc[mode] = errors("gru", ref_a, b200rnn.from_torch(ref_a).to(DEV).eval(), x)
    set_mode("ieee")
    # yardstick: stock torch.nn.GRU on CUDA, cuDNN at its default fp32 precision setting
    cudnn = torch.nn.GRU(256, 256, num_layers=2, batch_first=True).to(DEV).train()  # cuDNN backward needs train()
    cudnn.load_state_dict(ref_a.state_dict())
    acc["cudnn"] = errors("gru", ref_a, cudnn, x)
    acc["cudnn"]["cudnn_rnn_fp32_precision"] = torch.backends.cudnn.rnn.fp32_precision
    with torch.no_grad():
        res["cudnn_gru_fwd_ms"] = float(np.median([time_ms(lambda: cudnn(xa), args.iters) for _ in range(args.rounds)]))
    res["error_vs_fp64_gru_b128_t40"] = acc

    print(json.dumps(res, indent=1))
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
