"""A / B of two builds of the step library on the GPU: bit-identical outputs first, then alternating timed runs.

Both libraries are built into a temporary directory with the Makefile's flags: the base from another source tree (a directory holding
deepmimic_b200/csrc and include, or a git revision of this repository) and the branch from this tree.  For every workload, bench.py runs once
per build with --dump-outputs and every dumped array is compared with np.array_equal; then the timed runs alternate base / branch for the
remaining rounds (the dump runs are round 1).  The card's name, power limit and SM clocks are printed with the results.

  python tools/ab_step.py --base HEAD~1
  python tools/ab_step.py --base /path/to/parent/tree --workloads spinkick walk --rounds 3
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKLOADS = {"spinkick": "args/train_humanoid3d_spinkick_args.txt", "walk": "args/train_humanoid3d_walk_args.txt",
             "target_amp": "args/train_amp_target_humanoid3d_locomotion_args.txt", "dog_trot": "args/train_dog3d_trot_args.txt"}


def build(src_root, dst):
    """Copies src_root's deepmimic_b200/csrc and include to dst and builds dst/deepmimic_b200/libdeepmimic_b200.so there."""
    shutil.copytree(os.path.join(src_root, "deepmimic_b200", "csrc"), os.path.join(dst, "deepmimic_b200", "csrc"),
                    ignore=shutil.ignore_patterns("*.o", "*.so", "*.ptxas.log"))
    shutil.copytree(os.path.join(src_root, "include"), os.path.join(dst, "include"))
    csrc = os.path.join(dst, "deepmimic_b200", "csrc")
    subprocess.run(["make", "-j4", "../libdeepmimic_b200.so"], cwd=csrc, check=True, stdout=subprocess.DEVNULL)
    return os.path.join(dst, "deepmimic_b200", "libdeepmimic_b200.so")


def base_tree(base, tmp):
    if os.path.isdir(base):
        return base
    out = os.path.join(tmp, "base_src")
    os.makedirs(out)
    arc = subprocess.run(["git", "-C", REPO, "archive", base, "deepmimic_b200/csrc", "include"], check=True, stdout=subprocess.PIPE).stdout
    subprocess.run(["tar", "-x", "-C", out], input=arc, check=True)
    return out


def bench(lib, arg_file, a, dump=None):
    cmd = [sys.executable, os.path.join(REPO, "bench.py"), "--gpus", "1", "--steps", str(a.steps), "--warmup", str(a.warmup), "--no-cpu-baseline",
           "--arg-file", arg_file]
    if dump:
        cmd += ["--dump-outputs", dump]
    r = subprocess.run(cmd, cwd=REPO, env=dict(os.environ, DM_LIB=lib), check=True, stdout=subprocess.PIPE, text=True)
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="source tree of the base build, or a git revision of this repository")
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--rounds", type=int, default=3, help="timed runs per build and workload, the dump run included")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=4)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="ab_step_")
    try:
        libs = {"base": build(base_tree(a.base, tmp), os.path.join(tmp, "base")), "branch": build(REPO, os.path.join(tmp, "branch"))}
        print("card: name, power limit, max SM clock, SM clock:", card(), flush=True)
        runs = {w: {b: [] for b in libs} for w in a.workloads}
        identical = True
        for w in a.workloads:
            dumps = {}
            for b, lib in libs.items():
                dumps[b] = os.path.join(tmp, "dump", w, b)
                runs[w][b].append(bench(lib, WORKLOADS[w], a, dumps[b]))
            names = sorted(f for f in os.listdir(dumps["base"]) if f.endswith(".npy"))
            assert names == sorted(f for f in os.listdir(dumps["branch"]) if f.endswith(".npy")), "the builds dumped different arrays"
            diff = [n for n in names if not np.array_equal(np.load(os.path.join(dumps["base"], n)), np.load(os.path.join(dumps["branch"], n)))]
            identical &= not diff
            print("%-10s outputs %s (%s)" % (w, "bit-identical" if not diff else "DIFFER in " + ", ".join(diff), ", ".join(n[:-4] for n in names)), flush=True)
        for _ in range(a.rounds - 1):
            for w in a.workloads:
                for b, lib in libs.items():
                    runs[w][b].append(bench(lib, WORKLOADS[w], a))
        for w in a.workloads:
            for b in libs:
                rs = runs[w][b]
                print("%-10s %-6s policy_steps/s %s  kernel_ms %s  clocks %s" % (w, b, " ".join("%.4g" % r["value"] for r in rs),
                      " ".join("%.4f" % r["roofline"]["kernel_ms"] for r in rs), json.dumps(rs[-1].get("clocks"))), flush=True)
            lo, hi = min(r["value"] for r in runs[w]["branch"]), max(r["value"] for r in runs[w]["base"])
            print("%-10s branch / base (means) %.4f; slowest branch round %s every base round" % (
                w, np.mean([r["value"] for r in runs[w]["branch"]]) / np.mean([r["value"] for r in runs[w]["base"]]), "above" if lo > hi else "NOT above"), flush=True)
        print("card after the runs:", card())
        return 0 if identical else 1
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    sys.exit(main())
