"""A / B measurement of the moment kernel K1 against the library of another commit.

    python tools/bench_k1_ab.py build [--rev HEAD~1]        # compile <rev>'s libccab200.so (nvcc, no GPU needed)
    python tools/bench_k1_ab.py run [--rounds 5] [--out DIR] # on the GPU: alternate the two libraries

`build` exports <rev>'s CUDA sources with `git archive` into a temporary directory, compiles them with the same
Makefile and puts the library under build/k1_ab/ (ignored by git, so it stays out of the history and sits beside
the in-tree library).  `run` compares that library ("old") with the in-tree one ("new", as `__graft_entry__.build()`
left it).  Each round runs `bench.py --no-cpu --steps 20 --warmup 3` for `rcca` and `mcca4` once per library, in a
fresh subprocess that points `cca_zoo_b200._lib.LIB_PATH` at the library and runs bench.py through runpy; the order of
the two libraries alternates from round to round.  Then, once per library: `--dump-outputs` runs of `rcca` and `mcca4`
(weights and means compared bit for bit), the tf32x3b moment buffers of both inputs (compared with torch.equal) and one
`ccaloss512` run.  The card's name, power limit and maximum SM clock are read with a read-only nvidia-smi query.
`--parts` runs a subset.  The report is written as JSON under --out (a temporary directory unless given).
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OLD_DIR = os.path.join(ROOT, "build", "k1_ab", "old")
NEW_LIB = os.path.join(ROOT, "cca_zoo_b200", "libccab200.so")
OLD_LIB = os.path.join(OLD_DIR, "libccab200.so")

# bench.py under another library: the path is set before bench.py loads it
BENCH_CHILD = """
import runpy, sys
sys.path.insert(0, {root!r})
from cca_zoo_b200 import _lib
_lib.LIB_PATH = {lib!r}
sys.argv = ["bench.py"] + {args!r}
runpy.run_path({bench!r}, run_name="__main__")
"""

# the tf32x3b moment buffer of a bench.py input, saved as a torch file
MOMENTS_CHILD = """
import runpy, sys
sys.path.insert(0, {root!r})
from cca_zoo_b200 import _lib
_lib.LIB_PATH = {lib!r}
import torch
from cca_zoo_b200 import ops
b = runpy.run_path({bench!r}, run_name="bench_inputs")
b["W"].clear(); b["W"].update(b["WORKLOADS"][{workload!r}])
views = [torch.from_numpy(v).cuda() for v in b["make_views"](1000)]
torch.save(ops.moments(views, precision="tf32x3b").cpu(), {out!r})
"""


def build_old(rev: str) -> None:
    with tempfile.TemporaryDirectory() as tmp:
        arc = subprocess.run(["git", "-C", ROOT, "archive", rev, "cca_zoo_b200/csrc", "include"], check=True,
                             capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", tmp], input=arc, check=True)
        subprocess.run(["make", "-C", os.path.join(tmp, "cca_zoo_b200", "csrc"), "-j8"], check=True)
        os.makedirs(OLD_DIR, exist_ok=True)
        shutil.copy(os.path.join(tmp, "cca_zoo_b200", "libccab200.so"), OLD_LIB)
    sha = subprocess.run(["git", "-C", ROOT, "rev-parse", rev], check=True, capture_output=True, text=True).stdout
    with open(os.path.join(OLD_DIR, "REV"), "w") as f:
        f.write(sha)
    print(f"built {OLD_LIB} from {sha.strip()}")


def child(code: str) -> str:
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError(f"child failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
    return r.stdout


def bench(lib: str, args: list[str]) -> dict:
    out = child(BENCH_CHILD.format(root=ROOT, lib=lib, args=args, bench=os.path.join(ROOT, "bench.py")))
    lines = [ln for ln in out.splitlines() if ln.startswith("{")]
    return json.loads(lines[-1])


def pick(line: dict) -> dict:
    roof = line.get("roofline") or {}
    return {"ms_per_step": line["ms_per_step"], "kernel_ms": roof.get("kernel_ms"),
            "gpu_launches": line["gpu_launches"], "clocks": line.get("clocks")}


def same_npy(d0: str, d1: str) -> dict:
    import numpy as np

    names = sorted(n for n in os.listdir(d0) if n.endswith(".npy"))
    assert names == sorted(n for n in os.listdir(d1) if n.endswith(".npy")), "different output sets"
    res = {}
    for n in names:
        a, b = np.load(os.path.join(d0, n)), np.load(os.path.join(d1, n))
        res[n] = bool(a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b))
    return res


def run(rounds: int, outdir: str, parts: set) -> None:
    import torch

    os.makedirs(outdir, exist_ok=True)
    libs = {"old": OLD_LIB, "new": NEW_LIB}
    for name, path in libs.items():
        if not os.path.exists(path):
            raise RuntimeError(f"{name} library missing: {path}")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    report = {"gpu": smi, "old_rev": open(os.path.join(OLD_DIR, "REV")).read().strip() if
              os.path.exists(os.path.join(OLD_DIR, "REV")) else None, "rounds": []}
    timed = ["--no-cpu", "--steps", "20", "--warmup", "3"]
    for r in range(rounds if "timing" in parts else 0):
        order = ["old", "new"] if r % 2 == 0 else ["new", "old"]
        entry = {}
        for name in order:
            for wl in ("rcca", "mcca4"):
                entry[f"{name}/{wl}"] = pick(bench(libs[name], timed + ["--workload", wl]))
                print(f"round {r} {name:3s} {wl:6s} {json.dumps(entry[f'{name}/{wl}'])}", flush=True)
        report["rounds"].append(entry)

    summary = {}
    for name in libs if report["rounds"] else ():
        for wl in ("rcca", "mcca4"):
            for key in ("ms_per_step", "kernel_ms"):
                v = [e[f"{name}/{wl}"][key] for e in report["rounds"]]
                summary[f"{name}/{wl}/{key}"] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
            summary[f"{name}/{wl}/gpu_launches"] = sorted({e[f"{name}/{wl}"]["gpu_launches"] for e in report["rounds"]})
    report["summary"] = summary

    with tempfile.TemporaryDirectory() as tmp:
        same = {}
        for wl in ("rcca", "mcca4") if "bitwise" in parts else ():
            for name in libs:
                d = os.path.join(tmp, f"{name}_{wl}")
                bench(libs[name], timed + ["--workload", wl, "--dump-outputs", d])
                child(MOMENTS_CHILD.format(root=ROOT, lib=libs[name], bench=os.path.join(ROOT, "bench.py"),
                                           workload=wl, out=os.path.join(tmp, f"mom_{name}_{wl}.pt")))
            same[f"{wl}/outputs"] = same_npy(os.path.join(tmp, f"old_{wl}"), os.path.join(tmp, f"new_{wl}"))
            m0 = torch.load(os.path.join(tmp, f"mom_old_{wl}.pt"))
            m1 = torch.load(os.path.join(tmp, f"mom_new_{wl}.pt"))
            same[f"{wl}/moments_equal"] = bool(torch.equal(m0, m1))
        report["bitwise"] = same
    if "ccaloss" in parts:
        report["ccaloss512"] = {name: pick(bench(libs[name], timed + ["--workload", "ccaloss512"])) for name in libs}

    with open(os.path.join(outdir, f"k1_ab_{'_'.join(sorted(parts))}.json"), "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps({k: report.get(k) for k in ("gpu", "summary", "bitwise", "ccaloss512")}, indent=1))


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    b = sub.add_parser("build")
    b.add_argument("--rev", default="HEAD~1")
    r = sub.add_parser("run")
    r.add_argument("--rounds", type=int, default=5)
    r.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "k1_ab"))
    r.add_argument("--parts", default="timing,bitwise,ccaloss",
                   help="comma-separated subset of timing (the alternating rounds), bitwise, ccaloss")
    a = ap.parse_args()
    if a.cmd == "build":
        build_old(a.rev)
    else:
        run(a.rounds, a.out, set(a.parts.split(",")))


if __name__ == "__main__":
    main()
