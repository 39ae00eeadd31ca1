# coding: utf-8
"""Per-warp, per-phase cycle profile of engine 5's synthesis step (wn_kernel.cuh, WN_STAGE_PROF).

The shipped libwn.so has no counters.  This script compiles a profiling build of the same sources with
-DWN_STAGE_PROF into a temporary directory (or takes one with --lib), runs one synthesis call through it
(WN_LIB_PATH, WN_PROF=1; a first call warms up) and prints, per warp, the cycles each phase takes per stage:
mean over the blocks of the grid, with the smallest and largest block.  The counters cost registers and clock
reads of their own, so the profiled step is slower than the shipped one; compare profiles with each other.

    python scripts/stage_prof.py                       # config 2, T = 3000
    python scripts/stage_prof.py --lib /tmp/libwn_prof.so --json out.json
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from sweep import CFGS  # noqa: E402
from wavenet_vocoder_b200 import _native  # noqa: E402

SLOTS = 96                      # WN_PROF_SLOTS
NCRIT, NDEF = 13, 6             # counters per critical / deferred warp (WN_PC_CRIT, WN_PC_DEF)
SKEW, DEFB, TMA, COND = 52, 58, 82, 84   # WN_PS_SKEW, WN_PS_DEF, WN_PS_TMA, WN_PS_COND
CRIT = ["acquire+pre", "poll", "stash", "weight load+FMA issue", "wait for FMA results",
        "shuffle reduce", "quad_store", "barrier", "finalize", "publish", "wait for deferred"]
DEF = ["wait for stash", "unstash", "load+FMA+reduce+store", "barrier", "finalize"]


def build(out):
    cmd = _native.nvcc_command(out)
    cmd.insert(1, "-DWN_STAGE_PROF")
    print(" ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True)


def run(lib, cfg, T):
    env = dict(os.environ, WN_LIB_PATH=lib, WN_PROF="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "sweep.py"), "--child", cfg, str(T), "1", "1"],
                       env=env, capture_output=True, text=True, timeout=1200)
    if r.returncode != 0:
        raise SystemExit("profiled run failed:\n" + r.stderr[-3000:])
    rows = {}
    for ln in r.stderr.splitlines():       # wn_sync prints every call's counters: the last call wins
        if ln.startswith("WN_PROF_BLOCK"):
            f = ln.split()
            rows[int(f[1])] = [int(v) for v in f[2:]]
    if not rows:
        raise SystemExit("no WN_PROF_BLOCK lines: is %s a -DWN_STAGE_PROF build?" % lib)
    return np.array([rows[p] for p in sorted(rows)], dtype=np.float64), json.loads(r.stdout.strip().splitlines()[-1])


def cell(v):
    return "%.0f (%.0f–%.0f)" % (v.mean(), v.min(), v.max())


def report(pc, timing, cfg, T):
    L = CFGS[cfg]["layers"]
    ncs, nds = T * (L - 1), T * L          # critical stages 1..L-1; deferred stages 1..L
    out = {"cfg": cfg, "T": T, "us_per_step_profiled": timing["us_per_step"], "crit": {}, "deferred": {}}
    print("%s, T = %d, %d blocks; profiled step %.1f us (the counters slow it down)" %
          (cfg, T, pc.shape[0], timing["us_per_step"]))
    print("\ncritical group, cycles per stage of layers 1..L-1, mean over blocks (min–max block):\n")
    print("| phase | " + " | ".join("warp %d" % w for w in range(4)) + " |")
    print("|---|" + "---|" * 4)
    for i, name in enumerate(CRIT):
        cols = [pc[:, w * NCRIT + i] / ncs for w in range(4)]
        out["crit"][name] = [float(c.mean()) for c in cols]
        print("| %s | %s |" % (name, " | ".join(cell(c) for c in cols)))
    tot = [pc[:, w * NCRIT:w * NCRIT + len(CRIT)].sum(1) / ncs for w in range(4)]
    out["crit"]["stage total"] = [float(c.mean()) for c in tot]
    print("| stage total | %s |" % " | ".join(cell(c) for c in tot))
    for i, name in ((11, "stages 0, L + head, per step"), (12, "x_0 + step tail, per step")):
        cols = [pc[:, w * NCRIT + i] / T for w in range(4)]
        out["crit"][name] = [float(c.mean()) for c in cols]
        print("| %s | %s |" % (name, " | ".join(cell(c) for c in cols)))
    step = pc[:, 0:NCRIT].sum(1) / T
    out["crit"]["warp 0 step"] = float(step.mean())
    print("| warp 0, whole step | %s | | | |" % cell(step))
    skew = pc[:, SKEW] / np.maximum(pc[:, SKEW + 1], 1)
    last = pc[:, SKEW + 2:SKEW + 6] / np.maximum(pc[:, SKEW + 1:SKEW + 2], 1)
    out["skew"] = float(skew.mean())
    out["last_share"] = [float(v) for v in last.mean(0)]
    print("\narrival skew at the critical group's barrier (last - first warp): %s cycles per stage" % cell(skew))
    print("warp that arrives last: " + ", ".join("warp %d %.0f %%" % (w, 100 * last[:, w].mean()) for w in range(4)))
    print("\ndeferred group, cycles per deferred stage (layers 1..L), mean over blocks (min–max block):\n")
    print("| phase | " + " | ".join("warp %d" % (4 + w) for w in range(4)) + " |")
    print("|---|" + "---|" * 4)
    for i, name in enumerate(DEF):
        cols = [pc[:, DEFB + w * NDEF + i] / nds for w in range(4)]
        out["deferred"][name] = [float(c.mean()) for c in cols]
        print("| %s | %s |" % (name, " | ".join(cell(c) for c in cols)))
    cols = [pc[:, DEFB + w * NDEF + 5] / T for w in range(4)]
    out["deferred"]["pre-sums + step tail, per step"] = [float(c.mean()) for c in cols]
    print("| pre-sums + step tail, per step | %s |" % " | ".join(cell(c) for c in cols))
    for base, name in ((TMA, "TMA warp"), (COND, "conditioning warp")):
        wait, total = pc[:, base] / T, pc[:, base + 1] / T
        out[name] = {"wait_per_step": float(wait.mean()), "total_per_step": float(total.mean())}
        print("\n%s: waits %s of %s cycles per step" % (name, cell(wait), cell(total)), end="")
    print()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lib", help="a libwn.so built with -DWN_STAGE_PROF (default: build one in a temporary directory)")
    ap.add_argument("--cfg", default="cfg2", choices=sorted(CFGS))
    ap.add_argument("--T", type=int, default=3000)
    ap.add_argument("--json", help="also write the means to this file")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        lib = a.lib
        if lib is None:
            lib = os.path.join(tmp, "libwn_prof.so")
            build(lib)
        pc, timing = run(os.path.abspath(lib), a.cfg, a.T)
    out = report(pc, timing, a.cfg, a.T)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
