"""The default dispatch reaches each GRU H=256 forward config, and each runs forward and backward, fixed-length and ragged,
against stock torch CPU over T = 120 steps (the benchmark's length, so the error growth over a full sequence is covered).
The backward consumes the gates and n-gate pre-activations the forward kernel saves.

The dispatch tries the 4-CTA-cluster configs in the order bs2, bs4, tc8 and takes the first whose clusters are all
co-resident (an H100 SXM holds 30 four-CTA clusters; tc8 always runs):
  * B = 16: bs2 (8 clusters of 2 batch rows);
  * B = 96: bs4, since bs2 would need 48 clusters (24 of 4 rows);
  * B = 160: tc8, since bs4 would need 40 clusters, more than any H100 holds at once.
B200RNN_DEBUG prints one line per config the dispatch considered and is read once per process, so each case runs in a
child process."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BS2_LINE = "[b200rnn] fwd cfg C=4 BS=2 KL=16 UPL=8 RG=0 PB=0"
BS4_LINE = "[b200rnn] fwd cfg C=4 BS=4 KL=16 UPL=4 RG=1 PB=1"
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
spec = importlib.util.spec_from_file_location("gru256_fwd_configs", {path!r})
mod = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mod)
for ragged in (False, True):
    print("ERR", ragged, *mod._errors({B}, 120, ragged), flush=True)
"""


def _run_child(B):
    env = dict(os.environ, B200RNN_DEBUG="1")
    code = _CHILD.format(root=ROOT, pkg=os.path.join(ROOT, "icassp2022-depression_b200"), path=os.path.abspath(__file__),
                         B=B)
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    # one line per config the dispatch considered, in order; every launch considers bs2 first, and the last line before
    # the next launch is the config that ran
    cfgs = [ln.split(":")[0] for ln in proc.stderr.splitlines() if ln.startswith("[b200rnn] fwd cfg")]
    ran = [cfgs[i - 1] for i in range(1, len(cfgs) + 1) if i == len(cfgs) or cfgs[i] == BS2_LINE]
    errs = [[float(v) for v in ln.split()[2:]] for ln in proc.stdout.splitlines() if ln.startswith("ERR")]
    assert len(errs) == 2, proc.stdout + proc.stderr
    return cfgs, ran, errs, proc.stdout + proc.stderr


@pytest.mark.parametrize("B, line", [(16, BS2_LINE), (96, BS4_LINE), (160, TC8_LINE)], ids=["bs2_b16", "bs4_b96", "tc8_b160"])
def test_default_dispatch_reaches_config_t120(B, line):
    cfgs, ran, errs, out = _run_child(B)
    assert cfgs and cfgs[0] == BS2_LINE, cfgs
    assert ran and set(ran) == {line}, cfgs
    for err_y, err_dx, err_g in errs:
        assert err_y < 1e-5, out
        assert err_dx < 1e-4 and err_g < 1e-4, out
