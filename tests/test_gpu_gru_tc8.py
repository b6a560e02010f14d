"""The GRU H=256 forward config on the tensor cores (tc8: 8 batch rows per 4-CTA cluster, mma.sync m16n8k8 in 3xTF32),
fixed-length and ragged, forward and backward, against stock torch CPU over T = 120 steps (the benchmark's length, so the
error growth over a full sequence is covered). The backward consumes the gates and n-gate pre-activations the forward
kernel saves.

The config switch and the debug line are read once per process, so each case runs in a child process: with the config
forced (B200RNN_GRU_FWD=tc8) at the benchmark's B = 128, and through the default dispatch at B = 160, which needs 40
four-row clusters, more than any H100 holds at once, so the dispatch ends at tc8 whatever the chip's cluster capacity."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TC8_LINE = "[b200rnn] fwd cfg tc8 C=4 BS=8 mma.sync 3xTF32"


def _errors(B, T, ragged, seed=5):
    """max |y - y_ref|, |h_n - h_n_ref|; max |dx - dx_ref| / max |dx_ref|; max |dW - dW_ref| / max |dW_ref|"""
    import b200rnn

    torch.manual_seed(seed)
    ref = torch.nn.GRU(256, 256, num_layers=2, batch_first=True)
    mine = b200rnn.from_torch(ref).to(DEV)
    x = torch.randn(B, T, 256)
    lens = torch.randint(1, T + 1, (B,)) if ragged else torch.full((B,), T)
    lens[0] = T
    xr = x.clone().requires_grad_(True)
    xm = x.to(DEV).requires_grad_(True)
    outs = []
    for model, inp in ((ref, xr), (mine, xm)):
        if ragged:
            pk = torch.nn.utils.rnn.pack_padded_sequence(inp, lens, batch_first=True, enforce_sorted=False)
            y, h = model(pk)
            y = torch.nn.utils.rnn.pad_packed_sequence(y, batch_first=True, total_length=T)[0]
        else:
            y, h = model(inp)
        outs.append((y, h))
    (yr, hr), (ym, hm) = outs
    wy = torch.randn(B, T, 256)
    wh = torch.randn_like(hr)
    ((yr * wy).sum() + (hr * wh).sum()).backward()
    ((ym * wy.to(DEV)).sum() + (hm * wh.to(DEV)).sum()).backward()
    torch.cuda.synchronize()
    err_y = max((ym.detach().cpu() - yr.detach()).abs().max().item(), (hm.detach().cpu() - hr.detach()).abs().max().item())
    err_dx = ((xm.grad.cpu() - xr.grad).abs().max() / xr.grad.abs().max()).item()
    g_ref = torch.cat([p.grad.reshape(-1) for p in ref.parameters()])
    g_mine = torch.cat([p.grad.reshape(-1).cpu() for p in mine.parameters()])
    err_g = ((g_mine - g_ref).abs().max() / g_ref.abs().max()).item()
    return err_y, err_dx, err_g


_CHILD = """
import importlib.util, sys
sys.path[:0] = [{root!r}, {pkg!r}]
spec = importlib.util.spec_from_file_location("gru_tc8", {path!r})
mod = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mod)
for ragged in (False, True):
    print("ERR", ragged, *mod._errors({B}, 120, ragged), flush=True)
"""


def _run_child(B, extra_env):
    env = dict(os.environ)
    env.pop("B200RNN_GRU_FWD", None)
    env.update(B200RNN_DEBUG="1", **extra_env)
    code = _CHILD.format(root=ROOT, pkg=os.path.join(ROOT, "icassp2022-depression_b200"), path=os.path.abspath(__file__),
                         B=B)
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    # one line per config the dispatch considered, in order: the last one before each launch is the one that ran
    cfgs = [ln.split(":")[0] for ln in proc.stderr.splitlines() if ln.startswith("[b200rnn] fwd cfg")]
    errs = [[float(v) for v in ln.split()[2:]] for ln in proc.stdout.splitlines() if ln.startswith("ERR")]
    assert len(errs) == 2, proc.stdout + proc.stderr
    return cfgs, errs, proc.stdout + proc.stderr


@pytest.mark.parametrize("B, forced", [(128, True), (160, False)], ids=["forced_b128", "default_b160"])
def test_tc8_forward_backward_t120(B, forced):
    cfgs, errs, out = _run_child(B, {"B200RNN_GRU_FWD": "tc8"} if forced else {})
    assert cfgs and cfgs[-1] == TC8_LINE, cfgs
    if forced:
        assert set(cfgs) == {TC8_LINE}, cfgs
    assert not any("NG=2" in c for c in cfgs), cfgs   # bs8 is never taken by default
    for err_y, err_dx, err_g in errs:
        assert err_y < 1e-5, out
        assert err_dx < 1e-4 and err_g < 1e-4, out
