"""A/B timing of two builds of the library on bench.py's workload.

Runs R rounds, alternating the builds (A B, B A, A B, ...) so that drift of the shared machine falls on both, of

    bench.py --no-cpu-baseline --dump-outputs <tmp>/<build><round> [extra bench args]

each build selected through T4_LIB_PATH, and prints per run ms_per_step, the AssignRead pass's time (assign_pass.ms),
roofline.phase_share, extend_split, per_read and stream_balance, plus the stream kernel's device counters of the run
(bench.py's kernel-only launch).
Then it checks that every dumped .npy is byte-identical across all runs of both builds.

    python bench/ab_compare.py --build-parent HEAD       # cross-compile the parent into bench/_parent/ (git-ignored)
    python bench/ab_compare.py --a bench/_parent/libtrust4_b200.so --b trust4_b200/libtrust4_b200.so --rounds 3

The parent is compiled from `git archive <rev>` with __graft_entry__.NVCC_FLAGS, so it can be built where git is and
run from a copy of the tree that is not a repository.  Exit code 1 when the outputs differ.
"""
import argparse
import ctypes as C
import json
import os
import runpy
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARENT_DIR = os.path.join(ROOT, "bench", "_parent")
COUNTERS = {0: "reads", 1: "extend_dps", 16: "overlaps_extended", 20: "easy_reads", 21: "make_exact_calls", 22: "make_exact_cycles"}


def build_parent(rev):
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    os.makedirs(PARENT_DIR, exist_ok=True)
    out = os.path.join(PARENT_DIR, "libtrust4_b200.so")
    with tempfile.TemporaryDirectory() as src:
        archive = subprocess.run(["git", "-C", ROOT, "archive", rev], check=True, capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", src], input=archive, check=True)
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.run([nvcc] + g.NVCC_FLAGS + ["-o", out, os.path.join(src, "trust4_b200", "csrc", "t4_api.cu")], check=True)
    print("parent (%s) -> %s" % (rev, out))


def child(bench_args):
    """One bench.py run in this process, recording the counter snapshots bench.py takes around its kernel-only launch."""
    sys.path.insert(0, ROOT)
    from trust4_b200 import api
    lib = api.default_lib()
    real, snaps = lib.last_counters, []

    def last_counters(ptr):
        r = real(ptr)
        snaps.append(np.ctypeslib.as_array((C.c_uint64 * api.N_COUNTERS).from_address(ptr)).copy())
        return r
    lib.last_counters = last_counters
    sys.argv = ["bench.py"] + bench_args
    runpy.run_path(os.path.join(ROOT, "bench.py"), run_name="__main__")
    if len(snaps) >= 2:
        d = (snaps[-1] - snaps[-2]).astype(np.float64)
        print("AB_COUNTERS " + json.dumps({name: float(d[i]) for i, name in COUNTERS.items()}), flush=True)


def run_one(lib_path, dump_dir, bench_args):
    env = dict(os.environ, T4_LIB_PATH=os.path.abspath(lib_path))
    cmd = [sys.executable, os.path.abspath(__file__), "--child", "--", "--no-cpu-baseline", "--dump-outputs", dump_dir] + bench_args
    p = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-4000:] + p.stderr[-4000:])
        raise RuntimeError("bench.py failed with %s" % lib_path)
    line, ctr = None, None
    for s in p.stdout.splitlines():
        if s.startswith("AB_COUNTERS "):
            ctr = json.loads(s[len("AB_COUNTERS "):])
        elif s.startswith("{") and '"ms_per_step"' in s:
            line = json.loads(s)
    if line is None:
        raise RuntimeError("no bench line from %s" % lib_path)
    return line, ctr


def same_outputs(dirs):
    names = sorted(os.listdir(dirs[0]))
    bad = []
    for d in dirs[1:]:
        if sorted(os.listdir(d)) != names:
            bad.append((d, "file list"))
            continue
        for n in names:
            with open(os.path.join(dirs[0], n), "rb") as f0, open(os.path.join(d, n), "rb") as f1:
                if f0.read() != f1.read():
                    bad.append((d, n))
    return names, bad


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--build-parent", metavar="REV", help="cross-compile REV into bench/_parent/ and exit")
    ap.add_argument("--a", default=os.path.join(PARENT_DIR, "libtrust4_b200.so"), help="build A (default: the parent)")
    ap.add_argument("--b", default=os.path.join(ROOT, "trust4_b200", "libtrust4_b200.so"), help="build B (default: this tree's)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="", help="also write the runs and the summary as JSON here")
    ap.add_argument("bench_args", nargs="*", help="extra bench.py arguments (after --)")
    args = ap.parse_args()
    if args.child:
        return child(args.bench_args)
    if args.build_parent:
        return build_parent(args.build_parent)

    runs = []
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.rounds):
            order = [("A", args.a), ("B", args.b)] if r % 2 == 0 else [("B", args.b), ("A", args.a)]
            for name, path in order:
                d = os.path.join(tmp, "%s%d" % (name, r))
                line, ctr = run_one(path, d, args.bench_args)
                rl = line["roofline"]
                run = {"build": name, "round": r, "ms_per_step": line["ms_per_step"],
                       "assign_ms": (line.get("assign_pass") or {}).get("ms"), "phase_share": rl["phase_share"],
                       "extend_split": rl["extend_split"], "per_read": rl["per_read"], "stream_balance": rl["stream_balance"],
                       "counters": ctr, "dump": d}
                if ctr and ctr["reads"] > 0:
                    run["counters_per_read"] = {k: v / ctr["reads"] for k, v in ctr.items() if k != "reads"}
                runs.append(run)
                print(json.dumps({k: v for k, v in run.items() if k != "dump"}), flush=True)
        names, bad = same_outputs([x["dump"] for x in runs])

    ms = {b: [x["ms_per_step"] for x in runs if x["build"] == b] for b in ("A", "B")}
    ams = {b: [x["assign_ms"] for x in runs if x["build"] == b and x["assign_ms"] is not None] for b in ("A", "B")}
    summary = {"a": args.a, "b": args.b, "rounds": args.rounds,
               "ms_per_step": ms, "median_ms": {b: float(np.median(v)) for b, v in ms.items()},
               "b_vs_a_median": float(np.median(ms["B"]) / np.median(ms["A"]) - 1.0),
               "every_b_below_every_a": max(ms["B"]) < min(ms["A"]),
               "assign_ms": ams, "assign_median_ms": {b: float(np.median(v)) if v else None for b, v in ams.items()},
               "outputs_compared": names, "outputs_identical": not bad, "output_differences": bad}
    print("AB_SUMMARY " + json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ab_compare.json"), "w") as f:
            json.dump({"runs": [{k: v for k, v in x.items() if k != "dump"} for x in runs], "summary": summary}, f, indent=1)
    return 0 if not bad else 1


if __name__ == "__main__":
    sys.exit(main())
