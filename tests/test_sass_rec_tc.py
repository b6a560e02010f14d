"""Static check on the SASS of the tensor-core GRU forward recurrence (cuobjdump, no GPU): both instantiations
(fixed length and per-sequence lengths) run their contraction as HMMA.1688.F32.TF32 (mma.sync m16n8k8 tf32) and keep
every value in registers (no local-memory spill traffic)."""
import re
import shutil
import subprocess

import pytest

from b200rnn import _lib

cuobjdump = shutil.which("cuobjdump") or shutil.which("/usr/local/cuda/bin/cuobjdump")
pytestmark = pytest.mark.skipif(cuobjdump is None, reason="cuobjdump not available")


def _tc_kernels():
    txt = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    out, name = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "rec_fwd_tc_kernel" in m.group(1) else None
            if name:
                out[name] = []
        elif name is not None:
            m = re.search(r"\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                out[name].append(m.group(1))
    return out


def test_tc_recurrence_runs_on_hmma_without_spills():
    kernels = _tc_kernels()
    assert len(kernels) == 2, sorted(kernels)
    for name, ops in kernels.items():
        assert "HMMA.1688.F32.TF32" in ops, name
        spills = sorted({o for o in ops if o.startswith(("LDL", "STL"))})
        assert not spills, f"{name}: local-memory traffic {spills}"
