"""Two builds of the library, bit for bit: the forward outputs, every gradient and the launches of each backward call.

Each build runs the same seeded matrix in a process of its own (the build is chosen with B200RNN_LIB); the parent
process compares every tensor with torch.equal - the forward outputs y, h_n and c_n, dx, each dW / db, dh_0, dc_0,
dln_gamma / dln_beta and the gradient sinks' buffers - and the library launches per backward call (per call for the
no-grad cases). The workers run with B200RNN_DEBUG set and record per case the recurrence configs the library weighed
("[b200rnn] fwd cfg ...: need N clusters, capacity M, smem S"; the last line of each plan is the one that ran), so the
results show which configs ran and that both builds chose the same ones. The exit status is 0 only when every tensor,
every launch count and every config line (cluster capacities included) agree.

The cfg_* cases reach every config of the forward and backward plan tables (csrc/rnn_rec.cu plan_rec_fwd /
plan_rec_bwd), fixed-length and ragged, through the batch size: on an H100 with 66 two-CTA, 30 four-CTA and 15
eight-CTA co-resident clusters (DESIGN.md), GRU-256 runs 2-row clusters at B = 16, 4-row ones at B = 64 and tc8 /
8-CTA ones at B = 128; GRU-128 its 2-CTA config at B = 64 and the 4-CTA fallback at B = 272; the BiLSTM-256 its 4-CTA
config at B = 32 and the 8-CTA fallback at B = 64; the BiLSTM-128 its 2-CTA config at B = 16 and the 4-CTA fallback at
B = 136. The projected cases cover the four (H, P), the fused_nograd ones the fp16-pair forward of rnn_forward_fused.
The anyh_* cases run the runtime-sized kernels (csrc/rnn_anyh.cu) of the GRU, the LSTM and the Elman RNN (tanh and
relu), with W_hh on chip and read from L2, fixed-length with an initial state and ragged.

    # the other build, e.g. of an earlier commit, from a worktree of it:
    #   make -C <worktree>/icassp2022-depression_b200 OBJDIR=<tmp>/obj LIBDIR=$PWD/lib_parent
    python tools/bitwise.py --base lib_parent/libb200rnn.so [--out tools/bitwise_results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
sys.path[:0] = [ROOT, PKG]

DEV = "cuda:0"


def gpu_info():
    q = "name,power.limit,clocks.max.sm,driver_version"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock, driver = [s.strip() for s in out.split(",")]
    except Exception as e:  # noqa: BLE001
        name, power, clock, driver = "unknown", f"unknown ({e})", "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock, "driver": driver, "torch": torch.__version__}


# ---- worker: one build -----------------------------------------------------------------------------------------------

def _model(kind, I, H, L=2, bi=False, dropout=0.0, proj=0, seed=0):
    import b200rnn

    torch.manual_seed(seed)
    kw = {"proj_size": proj} if proj else {}
    if kind in ("rnn_tanh", "rnn_relu"):
        cls, kw = torch.nn.RNN, {"nonlinearity": kind[4:]}
    else:
        cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    ref = cls(I, H, num_layers=L, bidirectional=bi, batch_first=True, dropout=dropout, **kw)
    return b200rnn.from_torch(ref).to(DEV).train()


def _backward(loss):
    """library launches of loss.backward()"""
    from b200rnn import _lib

    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    loss.backward()
    torch.cuda.synchronize()
    return _lib.launch_count() - n0


def _weighted_sum(ts, seed):
    g = torch.Generator().manual_seed(seed)
    return sum((t * torch.randn(t.shape, generator=g).to(t.device)).sum() for t in ts)


def _run(m, B, T, *, hx=False, lengths=None, x_grad=True, seed=1):
    """y, h_n [, c_n], the gradients of sum(y * w1) + sum(h_n * w2) [+ sum(c_n * w3)] and the launches of its backward"""
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

    import b200rnn

    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, m.input_size, generator=g).to(DEV).requires_grad_(x_grad)
    h0 = None
    if hx:
        LD, HO = m.num_layers * (2 if m.bidirectional else 1), m.proj_size or m.hidden_size
        h0 = [0.5 * torch.randn(LD, B, HO, generator=g)]
        if isinstance(m, b200rnn.LSTM):  # (h_0, c_0)
            h0.append(0.5 * torch.randn(LD, B, m.hidden_size, generator=g))
        h0 = [h.to(DEV).requires_grad_(True) for h in h0]
    inp = x if lengths is None else pack_padded_sequence(x, lengths, batch_first=True, enforce_sorted=False)
    state0 = None if h0 is None else (tuple(h0) if len(h0) == 2 else h0[0])
    y, state = m(inp, state0)
    if lengths is not None:
        y = pad_packed_sequence(y, batch_first=True, total_length=T)[0]
    states = state if isinstance(state, tuple) else (state,)
    launches = _backward(_weighted_sum([y, *states], seed + 1))
    grads = {k: v.detach() for k, v in zip(("y", "h_n", "c_n"), (y, *states))}
    grads["dx"] = x.grad
    grads.update({"d" + n: p.grad for n, p in m.named_parameters()})
    for name, h in zip(("dh_0", "dc_0"), h0 or []):
        grads[name] = h.grad
    return grads, launches


def _misaligned_sink(m):
    """every weight gradient into a view one float past a 256-byte boundary, pre-filled (the kernels accumulate)"""
    params = list(m.parameters())
    offs, total = [], 0
    for p in params:
        offs.append(total + 1)
        total += (p.numel() + 1 + 63) // 64 * 64
    flat = 0.5 * torch.randn(total, generator=torch.Generator().manual_seed(7)).to(DEV)
    by_ptr = {p.data_ptr(): flat[o:o + p.numel()].view_as(p) for p, o in zip(params, offs)}
    m._grad_sink = lambda weights: [by_ptr[w.data_ptr()] for w in weights]
    return flat


def _ln_sum(m, B, T, seed=1):
    """forward_ln_sum under autograd: LayerNorm folded into layer 0 and the time sum into the last layer, both ways"""
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    ln = torch.nn.LayerNorm(m.input_size).to(DEV)
    with torch.no_grad():
        ln.weight.add_(0.1 * torch.randn(ln.weight.shape, generator=g).to(DEV))
        ln.bias.add_(0.1 * torch.randn(ln.bias.shape, generator=g).to(DEV))
    x = torch.randn(B, T, m.input_size, generator=g).to(DEV).requires_grad_(True)
    y = m.forward_ln_sum(x, ln)
    launches = _backward(_weighted_sum([y], seed + 1))
    grads = {"y": y.detach(), "dx": x.grad, "dln_gamma": ln.weight.grad, "dln_beta": ln.bias.grad}
    grads.update({"d" + n: p.grad for n, p in m.named_parameters()})
    return grads, launches


def _cases():
    """name -> callable returning (gradients, launches of the backward)"""
    import b200rnn

    def gru256(**kw):
        return _run(_model("gru", 256, 256), 64, 120, **kw)

    def bilstm256_ragged():
        lens = torch.randint(1, 31, (32,), generator=torch.Generator().manual_seed(3))
        lens[0] = 30
        return _run(_model("lstm", 1024, 256, bi=True), 32, 30, lengths=lens)

    def frozen_w_ih():
        m = _model("gru", 256, 256)
        m.weight_ih_l0.requires_grad_(False)
        return _run(m, 64, 120)

    def grad_bucket():
        m = _model("gru", 256, 256)
        bucket = b200rnn.GradBucket(m)
        grads, n = _run(m, 64, 120)
        return {**grads, "bucket": bucket.flat}, n

    def misaligned(kind, H, bi):
        m = _model(kind, 256, H, bi=bi)
        flat = _misaligned_sink(m)
        grads, n = _run(m, 32, 40)
        return {**grads, "sink": flat}, n

    cases = {
        "gru256_i256_l2_b64_t120": gru256,
        "gru128_i40_dropout0.3_b64_t50": lambda: _run(_model("gru", 40, 128, dropout=0.3), 64, 50),
        "bilstm256_i1024_packed_ragged_b32_t30": bilstm256_ragged,
        "bilstm128_i256_hx_b16_t40": lambda: _run(_model("lstm", 256, 128, bi=True), 16, 40, hx=True),
        "gru256_i256_hx_t1_b16": lambda: _run(_model("gru", 256, 256), 16, 1, hx=True),
        "lstmp_h256_p64_i256_l2_d2_b16_t40": lambda: _run(_model("lstm", 256, 256, bi=True, proj=64), 16, 40,
                                                          hx=True),
        "grad_bucket_gru256_b64_t120": grad_bucket,
        "misaligned_sink_gru256_b32_t40": lambda: misaligned("gru", 256, False),
        "misaligned_sink_bilstm128_b32_t40": lambda: misaligned("lstm", 128, True),
        "frozen_weight_ih_l0_gru256_b64_t120": frozen_w_ih,
        "input_without_grad_gru256_b64_t120": lambda: gru256(x_grad=False),
        "forward_ln_sum_gru256_i256_b64_t120": lambda: _ln_sum(_model("gru", 256, 256), 64, 120),
    }
    def ragged(B, T):
        lens = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(3))
        lens[0] = T
        return lens

    def cfg_case(kind, I, H, B, bi, proj=0, packed=False, T=24, hx=None):
        return lambda: _run(_model(kind, I, H, bi=bi, proj=proj), B, T, hx=proj > 0 if hx is None else hx,
                            lengths=ragged(B, T) if packed else None)

    matrix = [("gru", 256, 256, B, False, 0) for B in (16, 64, 128)]
    matrix += [("gru", 40, 128, B, False, 0) for B in (64, 272)]
    matrix += [("lstm", 256, 256, B, True, 0) for B in (32, 64)]
    matrix += [("lstm", 256, 128, B, True, 0) for B in (16, 136)]
    matrix += [("lstm", 256, H, 16, True, P) for H, P in ((128, 32), (128, 64), (256, 64), (256, 128))]
    for kind, I, H, B, bi, P in matrix:
        for packed in (False, True):
            name = f"cfg_{'bi' if bi else ''}{kind}{H}{f'_p{P}' if P else ''}_i{I}_b{B}_t24{'_ragged' if packed else ''}"
            cases[name] = cfg_case(kind, I, H, B, bi, P, packed)

    # The runtime-sized kernels (csrc/rnn_anyh.cu), each shape fixed-length with an initial state and ragged without:
    # GRU / LSTM at hidden sizes without a fixed config, W_hh on chip (GRU 64, BiLSTM 192) and read from L2 (GRU 1024,
    # LSTM 768), and the Elman RNN on chip (tanh 128, relu 512) and from L2 (tanh 1024)
    anyh = [("gru", 40, 64, 64, False), ("lstm", 40, 192, 16, True), ("gru", 40, 1024, 8, False),
            ("lstm", 40, 768, 8, False), ("rnn_tanh", 40, 128, 64, False), ("rnn_relu", 40, 512, 64, False),
            ("rnn_tanh", 40, 1024, 8, False)]
    for kind, I, H, B, bi in anyh:
        for packed in (False, True):
            name = f"anyh_{'bi' if bi else ''}{kind}{H}_i{I}_b{B}_t24{'_ragged' if packed else '_hx'}"
            cases[name] = cfg_case(kind, I, H, B, bi, packed=packed, hx=not packed)

    def fused_nograd(pool_sum):
        from b200rnn import _lib
        from b200rnn.functional import rnn_forward_fused

        m = _model("gru", 256, 256)
        x = torch.randn(160, 40, 256, generator=torch.Generator().manual_seed(5)).to(DEV)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        with torch.no_grad():
            out, h_n = rnn_forward_fused(x, m._flat_weights, m._config(), pool_sum=pool_sum)[:2]
        torch.cuda.synchronize()
        return {"y_pool" if pool_sum else "y": out, "h_n": h_n}, _lib.launch_count() - n0

    cases["fused_nograd_gru256_i256_l2_b160_t40"] = lambda: fused_nograd(False)
    cases["fused_nograd_pool_sum_gru256_i256_l2_b160_t40"] = lambda: fused_nograd(True)

    for name in ("gru256_i256_l2_b64_t120", "bilstm256_i1024_packed_ragged_b32_t30", "cfg_gru256_i256_b128_t24",
                 "cfg_gru256_i256_b128_t24_ragged"):
        fn = cases[name]

        def tf32(fn=fn):
            torch.backends.cuda.matmul.fp32_precision = "tf32"
            try:
                return fn()
            finally:
                torch.backends.cuda.matmul.fp32_precision = "ieee"
        cases["tf32_" + name] = tf32
    return cases


def _configs(fn):
    """fn() with fd 2 captured: its result and the B200RNN_DEBUG config lines the library printed, in order"""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile() as f:
        os.dup2(f.fileno(), 2)
        try:
            res = fn()
            torch.cuda.synchronize()
        finally:
            sys.stderr.flush()
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        lines = f.read().decode(errors="replace").splitlines()
    return res, list(dict.fromkeys(l for l in lines if l.startswith("[b200rnn]")))


def worker(out):
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    res = {}
    for name, fn in _cases().items():
        (grads, launches), configs = _configs(fn)
        res[name] = {"grads": {k: (None if v is None else v.detach().cpu()) for k, v in grads.items()},
                     "launches": launches, "configs": configs}
    torch.save(res, out)


# ---- driver: both builds, compared -----------------------------------------------------------------------------------

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default=os.path.join(ROOT, "lib_parent", "libb200rnn.so"),
                    help="the build to compare against")
    ap.add_argument("--lib", default=os.path.join(PKG, "lib", "libb200rnn.so"), help="the build under test")
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "bitwise_results.json"))
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.worker)

    runs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for tag, lib in (("base", args.base), ("new", args.lib)):
            path = os.path.join(tmp, tag + ".pt")
            env = dict(os.environ, B200RNN_LIB=os.path.abspath(lib), B200RNN_DEBUG="1")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", path], env=env, check=True)
            runs[tag] = torch.load(path)
    cases, all_equal, launches_equal, configs_equal = {}, True, True, True
    for name, base in runs["base"].items():
        new = runs["new"][name]
        diff = [k for k, v in base["grads"].items()
                if (v is None) != (new["grads"][k] is None) or (v is not None and not torch.equal(v, new["grads"][k]))]
        computed = [k for k, v in base["grads"].items() if v is not None]
        fwd = [k for k in computed if k in ("y", "y_pool", "h_n", "c_n")]
        cases[name] = {"forward": fwd, "gradients": sorted(k for k in computed if k not in fwd),
                       "not_computed": sorted(k for k, v in base["grads"].items() if v is None),
                       "bit_identical": not diff and base["grads"].keys() == new["grads"].keys(), "differ": diff,
                       "launches_base": base["launches"], "launches_new": new["launches"],
                       "configs": new["configs"], "configs_equal": base["configs"] == new["configs"]}
        all_equal &= cases[name]["bit_identical"]
        launches_equal &= base["launches"] == new["launches"]
        configs_equal &= cases[name]["configs_equal"]
    res = {"device": gpu_info(), "all_bit_identical": all_equal, "launches_equal": launches_equal,
           "configs_equal": configs_equal, "cases": cases}
    print(json.dumps(res, indent=1))
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
        f.write("\n")
    return 0 if all_equal and launches_equal and configs_equal else 1


if __name__ == "__main__":
    sys.exit(main())
