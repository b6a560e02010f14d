"""Do the numerics tests bite? Build the library with one small arithmetic mutation at a time and run the tests on it.

Each mutation is one textual edit of csrc/ that changes arithmetic only - no indexing, barrier or memory access - and is
applied to a copy of the sources in a temporary directory; that copy is built (make, as build() does) and loaded with
B200RNN_LIB. Against each build the script runs tests/test_gpu_numerics_f64.py and the existing GPU numerics tests, and
records per mutation which tests fail. A mutation that no new test catches is a hole in the suite.

    python tools/numerics_mutants.py [--only NAME ...] [--out tools/numerics_mutants_results.json]
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
sys.path[:0] = [ROOT, PKG]

# name -> (file under csrc/, text, replacement, what it breaks)
MUTATIONS = {
    "x3_drop_ah_bl": ("rnn_rec.cu", "            ptx::mma_tf32_m16n8k8(d[g][0], ah, bl);\n", "",
                      "3xTF32 tc8 recurrence: the hi(W) * lo(h) correction mma is lost"),
    "f16_drop_ah_bl": ("rnn_rec.cu", "            ptx::mma_f16_m16n8k16(d[g][0], ah, bl);\n", "",
                       "fp16-pair tc8 recurrence: the hi(W) * lo(h) correction mma is lost"),
    "fwdcell_drop_bhn": ("rnn_rec.cu", "const float hn = pre[2] + bhn;", "const float hn = pre[2];",
                         "every GRU forward config: b_hn left out of the candidate gate"),
    "bwd_drop_one_minus_r": ("rnn_rec.cu", "const float dr = dn * hn * r * (1.f - r);", "const float dr = dn * hn * r;",
                             "GRU BPTT: the sigmoid derivative of r loses its (1 - r) factor"),
}
NEW = "tests/test_gpu_numerics_f64.py"
EXISTING = ["tests/test_gpu_parity.py", "tests/test_gpu_property.py", "tests/test_gpu_coverage.py",
            "tests/test_gpu_varlen.py", "tests/test_gpu_proj.py", "tests/test_gpu_h16_fwd.py"]


def gpu_info():
    q = "name,power.limit,clocks.max.sm,driver_version"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock, driver = [s.strip() for s in out.split(",")]
    except Exception as e:  # noqa: BLE001
        name, power, clock, driver = "unknown", f"unknown ({e})", "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock, "driver": driver}


def build(tmp, name):
    """the mutated library: copies of csrc/, the Makefile and include/ under tmp, one edit, make"""
    src, before, after, _ = MUTATIONS[name]
    pkg = os.path.join(tmp, name, "pkg")
    shutil.copytree(os.path.join(PKG, "csrc"), os.path.join(pkg, "csrc"))
    shutil.copy(os.path.join(PKG, "Makefile"), pkg)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, name, "include"))
    path = os.path.join(pkg, "csrc", src)
    text = open(path).read()
    if text.count(before) != 1:
        raise SystemExit(f"{name}: the text to mutate occurs {text.count(before)} times in {src}")
    with open(path, "w") as f:
        f.write(text.replace(before, after))
    jobs = str(max(1, min(8, os.cpu_count() or 1)))
    subprocess.run(["make", "-C", pkg, "-j", jobs], check=True, capture_output=True)
    return os.path.join(pkg, "lib", "libb200rnn.so")


def failing(lib, paths, maxfail=None):
    """ids of the tests in `paths` that fail (or error) against the library `lib`"""
    env = dict(os.environ, B200RNN_LIB=lib)
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-rfE", "--tb=no", *paths]
    if maxfail:
        cmd.append(f"--maxfail={maxfail}")
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True).stdout
    return sorted(set(re.findall(r"^(?:FAILED|ERROR) (\S+)", out, re.M)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", nargs="*", choices=list(MUTATIONS))
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "numerics_mutants_results.json"))
    args = ap.parse_args()
    res = {"mutations": {}}
    if os.path.exists(args.out):   # a run of some mutations (--only) adds to the results of the others
        with open(args.out) as f:
            res = json.load(f)
    res["device"] = gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        for name in args.only or MUTATIONS:
            lib = build(tmp, name)
            new = failing(lib, [NEW])
            old = {p: failing(lib, [p], maxfail=1) for p in EXISTING}
            res["mutations"][name] = {
                "file": MUTATIONS[name][0], "replaced": MUTATIONS[name][1].strip(),
                "with": MUTATIONS[name][2].strip(), "breaks": MUTATIONS[name][3],
                "new_tests_failing": new, "caught_by_new_tests": bool(new),
                "existing_first_failure": {p: f[0] for p, f in old.items() if f},
                "caught_by_existing_tests": any(old.values()),
            }
            print(name, "new:", len(new), "existing:", res["mutations"][name]["caught_by_existing_tests"], flush=True)
            with open(args.out, "w") as f:   # after each mutation: a long run keeps what it has measured
                json.dump(res, f, indent=1)
                f.write("\n")
    return 0 if all(m["caught_by_new_tests"] for m in res["mutations"].values()) else 1


if __name__ == "__main__":
    sys.exit(main())
