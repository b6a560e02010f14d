#!/usr/bin/env python
"""Per-launch time of the input-projection GEMM at the fuse step's forward shapes (library profile hook, CUDA events).

For each shape it times, alone on the card:
  * `presplit`: the generic GEMM entry (b200rnn_gemm_f32). The A split pass is a separate launch and is not counted:
    this is the GEMM kernel as the forward ran it before A was split on chip;
  * `f32a`: the fp32-A GEMM (3xTF32, A split in registers), when the loaded library has it;
  * `f16a`: the fp16-pair fp32-A GEMM of the no-grad fused forward, when the loaded library has it.
and beside the recurrence: the audio GRU branch (2 streamed layers) at B = 128, as bench.py's roofline pass does.
The per-tile cost outside the k-loop (epilogue, tile switch) is estimated from the audio shape at K = 256 and K = 512:
t(K) = waves * (k-blocks * c + e), so e = (2 t(256) - t(512)) / waves.
MMA TFLOP/s counts the 3 TF32 products; bytes are what the kernel has to move, computed from the shapes (A once per
column tile, W presplit once per row tile, C written once).

    python tools/gemm_launch_times.py [--reps 50]      # B200RNN_LIB=... to time another build of the library
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "icassp2022-depression_b200"))

import torch  # noqa: E402

import b200rnn  # noqa: E402
from b200rnn import _lib  # noqa: E402

SHAPES = {"audio_layer": (15360, 768, 256), "text_layer0_dir": (3840, 512, 1024)}


def _profiled(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    _lib.profile(True)
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    ms, n = _lib.profile_read(_lib.PROF_GEMM)
    _lib.profile(False)
    return ms / max(n, 1), n


def _bytes(M, N, K, a_bytes_per_elem):
    tiles_m, tiles_n = (M + 127) // 128, N // 128
    return tiles_n * M * K * a_bytes_per_elem + tiles_m * N * K * 8 + M * N * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = _lib.load()
    f32a = getattr(lib, "b200rnn_debug_gemm_f32a", None)
    out = {"device": torch.cuda.get_device_name(dev), "library": _lib.LIB_PATH, "alone": {}}
    g = torch.Generator().manual_seed(0)
    for name, (M, N, K) in SHAPES.items():
        A = torch.randn(M, K, generator=g).to(dev)
        W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        C = torch.empty(M, N, device=dev)
        flops = 3 * 2 * M * N * K
        res = {}
        ms, n = _profiled(lambda: b200rnn.gemm(A, W, bias=bias, out=C), args.reps)
        res["presplit"] = {"ms": ms, "launches": n, "mma_tflops": flops / ms / 1e9,
                           "bytes": _bytes(M, N, K, 8), "gb_s": _bytes(M, N, K, 8) / ms / 1e6}
        if f32a is not None:
            import ctypes

            f32a.restype = ctypes.c_int
            f32a.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int] + \
                [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
            sbytes = 8 * (M + N) * K + 4096
            scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream

            def run():
                _lib.check(f32a(M, N, K, A.data_ptr(), K, 0, 0, W.data_ptr(), C.data_ptr(), bias.data_ptr(), None, 0,
                                scratch.data_ptr(), sbytes, stream), "debug_gemm_f32a")

            ms, n = _profiled(run, args.reps)  # includes the per-call W split launch only in PROF_MISC
            res["f32a"] = {"ms": ms, "launches": n, "mma_tflops": flops / ms / 1e9,
                           "bytes": _bytes(M, N, K, 4), "gb_s": _bytes(M, N, K, 4) / ms / 1e6}
            f16a = getattr(lib, "b200rnn_debug_gemm_f16a", None)
            if f16a is not None:  # the fp16-pair kernel of the no-grad fused forward (W split per call: PROF_MISC)
                f16a.restype, f16a.argtypes = f32a.restype, f32a.argtypes

                def run16():
                    _lib.check(f16a(M, N, K, A.data_ptr(), K, 0, 0, W.data_ptr(), C.data_ptr(), bias.data_ptr(), None,
                                    0, scratch.data_ptr(), sbytes, stream), "debug_gemm_f16a")

                ms16, n16 = _profiled(run16, args.reps)
                res["f16a"] = {"ms": ms16, "launches": n16, "vs_f32a": ms16 / ms}
        out["alone"][name] = {"M": M, "N": N, "K": K, **res}
        if f32a is not None and name == "audio_layer":
            t1 = res["f32a"]["ms"]
            K2 = 2 * K
            A = torch.randn(M, K2, generator=g).to(dev)
            W = (torch.randn(N, K2, generator=g) / K2 ** 0.5).to(dev)
            sbytes = 8 * (M + N) * K2 + 4096
            scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)

            def run2():
                _lib.check(f32a(M, N, K2, A.data_ptr(), K2, 0, 0, W.data_ptr(), C.data_ptr(), bias.data_ptr(), None,
                                0, scratch.data_ptr(), sbytes, stream), "debug_gemm_f32a")

            t2, _ = _profiled(run2, args.reps)
            waves = ((M + 127) // 128) * (N // 128) / torch.cuda.get_device_properties(dev).multi_processor_count
            e_us = (2 * t1 - t2) / waves * 1e3
            c_us = (t2 - t1) / waves / (K // 32) * 1e3
            out["alone"][name]["f32a_tile_split"] = {"ms_at_K512": t2, "kblock_us": c_us, "outside_kloop_us": e_us,
                                                     "outside_share": e_us / (e_us + (K // 32) * c_us)}
    # beside the recurrence: the streamed audio GRU, 2 layers, B = 128, T = 120, eval
    torch.manual_seed(0)
    gru = b200rnn.from_torch(torch.nn.GRU(256, 256, num_layers=2, batch_first=True)).to(dev).eval()
    x = torch.randn(128, 120, 256, device=dev)
    with torch.no_grad():
        ms, n = _profiled(lambda: gru(x), args.reps)
    out["beside_recurrence"] = {"audio_gru_2_layers_B128_T120": {"gemm_ms_per_launch": ms, "launches": n}}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
