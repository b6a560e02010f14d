"""The GRU H=256 forward config with 8 batch rows per 4-CTA cluster (`<4,8,16,2,0>`, two unit groups per warp, 8 warps
per CTA) and its per-sequence-length twin, against stock torch CPU.

B = 160 needs 40 four-CTA clusters of 4 rows, more than any H100 holds at once, so the dispatch takes the 8-row config
whatever the chip's cluster capacity. At B = 128 the dispatch may prefer another config, so that size runs in a child
process with the config forced (B200RNN_GRU_FWD=bs8, read once per process) and B200RNN_DEBUG=1 showing which config
ran."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _forward_error(B, T, ragged, seed=11):
    import b200rnn

    torch.manual_seed(seed)
    ref = torch.nn.GRU(256, 256, num_layers=2, batch_first=True)
    mine = b200rnn.from_torch(ref).to(DEV)
    x = torch.randn(B, T, 256)
    with torch.no_grad():
        if ragged:
            lens = torch.randint(1, T + 1, (B,))
            lens[0] = T
            pk = lambda t: torch.nn.utils.rnn.pack_padded_sequence(t, lens, batch_first=True, enforce_sorted=False)  # noqa: E731
            yr, hr = ref(pk(x))
            ym, hm = mine(pk(x.to(DEV)))
            yr = torch.nn.utils.rnn.pad_packed_sequence(yr, batch_first=True, total_length=T)[0]
            ym = torch.nn.utils.rnn.pad_packed_sequence(ym, batch_first=True, total_length=T)[0]
        else:
            yr, hr = ref(x)
            ym, hm = mine(x.to(DEV))
    torch.cuda.synchronize()
    return max((ym.cpu() - yr).abs().max().item(), (hm.cpu() - hr).abs().max().item())


@pytest.mark.parametrize("ragged", [False, True])
def test_bs8_config_beyond_the_4_row_capacity(ragged):
    assert _forward_error(160, 12, ragged) < 1e-5


_CHILD = """
import importlib.util, sys
sys.path[:0] = [{root!r}, {pkg!r}]
spec = importlib.util.spec_from_file_location("gru_bs8_clusters", {path!r})
mod = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mod)
for ragged in (False, True):
    print("ERR", ragged, mod._forward_error(128, 20, ragged), flush=True)
"""


def test_bs8_config_forced_at_b128():
    env = dict(os.environ, B200RNN_GRU_FWD="bs8", B200RNN_DEBUG="1")
    code = _CHILD.format(root=ROOT, pkg=os.path.join(ROOT, "icassp2022-depression_b200"), path=os.path.abspath(__file__))
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    cfgs = {ln.split(":")[0] for ln in proc.stderr.splitlines() if ln.startswith("[b200rnn] fwd cfg")}
    assert cfgs == {"[b200rnn] fwd cfg C=4 BS=8 KL=16 UPL=2 RG=0 PB=0 NG=2"}, proc.stderr
    errs = [float(ln.split()[2]) for ln in proc.stdout.splitlines() if ln.startswith("ERR")]
    assert len(errs) == 2 and max(errs) < 1e-5, proc.stdout
