"""Every recurrence kernel compiles without stack and without local memory (cuobjdump -res-usage of the built library).

The kernels keep their state, weights and accumulators in registers across the whole step loop, and all the helpers
they share (the cluster slice, the exchange barriers, the LSTM cell) are force-inlined: a spill or a stack frame would
put local-memory traffic on the serial path of every step."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "icassp2022-depression_b200", "lib", "libb200rnn.so")


def _rec_kernels():
    """(STACK, LOCAL) of every rec_* kernel, by mangled name"""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    seen, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and name and re.search(r"\d(rec_\w+_kernel)I", name):
            seen[name] = (int(m.group(1)), int(m.group(2)))
    return seen


def test_recurrence_kernels_use_no_local_memory_and_no_stack():
    seen = _rec_kernels()
    # FFMA forward 16, tc8 forward 6 (3xTF32, TF32, fp16 pairs), FFMA backward 18, projected 16; each fixed-length and VL
    assert len(seen) == 56, sorted(seen)
    assert len([n for n in seen if "_proj_" in n]) == 16, sorted(seen)
    assert all(v == (0, 0) for v in seen.values()), {n: v for n, v in seen.items() if v != (0, 0)}
