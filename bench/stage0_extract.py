#!/usr/bin/env python3
"""Stage 0 end to end: the stock `fastq-extractor` against the drop-in `fastq-extractor-gpu` on one synthetic read set.

    python bench/stage0_extract.py [--pairs 2000000] [--formats fq,gz] > stage0_extract.json

Writes 150 bp pairs with a fixed seed into a temporary directory (90 % random decoys, the share of a bulk RNA-seq library
that does not come from an immune receptor; the rest windows of synthetic clonotypes, tests/extractor_cases.py), as plain
.fq and as .fq.gz, and runs both binaries (oracle/_ref/, as the build left them) at -t 1 and at -t = all host cores,
each with its own output prefix.  One JSON line: wall time and reads/s of every run, the drop-in's own split of its wall
time into the gene-set upload, the device scan (t4_refset_scan calls: copies, launch and wait) and the rest (host FASTQ
parsing, the worker threads' replay and the output), whether every output file equals the stock binary's, which side
bounds the drop-in, and the card name, power limit and host core count read in the same call."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = os.path.join(ROOT, "oracle", "_ref")
LINE = re.compile(r"stage-0 route: (\d+) reads scanned on the device, (\d+) on the host \((\d+) batches; gene set ([\d.]+) s, "
                  r"device scan ([\d.]+) s\)")


def card():
    """Name and power limit of the first card (a read-only nvidia-smi query)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    except OSError:
        return {"name": None, "power_limit": None}
    if q.returncode != 0 or not q.stdout.strip():
        return {"name": None, "power_limit": None}
    name, pl = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
    return {"name": name, "power_limit": pl}


def run(exe, args, prefix, threads):
    t0 = time.perf_counter()
    r = subprocess.run([exe, "-t", str(threads), "-o", prefix] + args, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)
    wall = time.perf_counter() - t0
    if r.returncode != 0:
        sys.exit("%s failed (%d): %s" % (exe, r.returncode, r.stderr[-2000:]))
    return wall, r.stderr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2000000)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--decoy", type=float, default=0.9)
    ap.add_argument("--formats", default="fq,gz")
    a = ap.parse_args()
    import extractor_cases as xc
    stock, dropin = os.path.join(REF, "fastq-extractor"), os.path.join(REF, "fastq-extractor-gpu")
    for exe in (stock, dropin):
        if not os.path.exists(exe):
            sys.exit("%s not built (python -c 'import __graft_entry__ as g; g.build()' where the reference sources are present)" % exe)
    cores = os.cpu_count() or 1
    out = {"what": "fastq-extractor end to end: stock binary vs the drop-in whose candidate test is t4_refset_scan on the device",
           "pairs": a.pairs, "read_len": 150, "decoy_fraction": a.decoy, "seed": a.seed, "card": card(), "host_cores": cores,
           "runs": []}
    tmp = tempfile.mkdtemp(prefix="t4s0x")
    try:
        fa = xc.gene_fasta(os.path.join(tmp, "genes.fa"))
        t0 = time.perf_counter()
        inputs = {}
        for fmt in a.formats.split(","):
            ext = ".fq.gz" if fmt == "gz" else ".fq"
            f1, f2 = os.path.join(tmp, "r_1" + ext), os.path.join(tmp, "r_2" + ext)
            xc.write_bulk_fastq(f1, f2, a.seed, a.pairs, 150, a.decoy, gz=(fmt == "gz"))
            inputs[fmt] = ["-f", fa, "-1", f1, "-2", f2]
        out["generate_s"] = time.perf_counter() - t0
        reads = 2 * a.pairs
        for fmt, args in inputs.items():
            for threads in sorted({1, cores}):
                rec = {"format": fmt, "threads": threads}
                files = {}
                for tag, exe in (("stock", stock), ("gpu", dropin)):
                    pre = os.path.join(tmp, "%s_%s_t%d" % (tag, fmt, threads))
                    wall, err = run(exe, args, pre, threads)
                    rec[tag] = {"wall_s": wall, "reads_per_s": reads / wall}
                    if tag == "gpu":
                        m = LINE.search(err)
                        if not m:
                            sys.exit("the drop-in printed no route line: " + err[-2000:])
                        dev, host, batches, gs, scan = int(m.group(1)), int(m.group(2)), int(m.group(3)), float(m.group(4)), float(m.group(5))
                        rec[tag].update({"device_reads": dev, "host_reads": host, "batches": batches, "gene_set_s": gs,
                                         "device_scan_s": scan, "host_parse_output_s": wall - gs - scan,
                                         "device_scan_reads_per_s": dev / scan if scan > 0 else None})
                    files[tag] = {suf: open(pre + suf, "rb").read() for suf in ("_1.fq", "_2.fq")}
                rec["outputs_equal"] = files["stock"] == files["gpu"]
                rec["kept_pairs"] = files["stock"]["_1.fq"].count(b"\n") // 4
                rec["speedup"] = rec["stock"]["wall_s"] / rec["gpu"]["wall_s"]
                g = rec["gpu"]
                rec["gpu_bound_by"] = "host FASTQ parsing and output" if g["host_parse_output_s"] > g["device_scan_s"] else "device scan"
                out["runs"].append(rec)
                for f in os.listdir(tmp):
                    if f.startswith(("stock_", "gpu_")):
                        os.remove(os.path.join(tmp, f))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    out["all_outputs_equal"] = all(r["outputs_equal"] for r in out["runs"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
