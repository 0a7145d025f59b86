"""Hits per c_get_hits call during the run, and how many bits of the (strand | contig | diagonal) prefix vary per read.

bench.py reports only the mean (counter 4 over reads).  This drives a uniform sample of the bench workload's streams
through the per-call API: before each record's AddRead it fetches the read's hits with t4_seqset_get_hits on the set
as it is at that point, then runs the record alone through t4_seqset_add_reads_batch.  Records run one at a time have
no mate or run-of-identical-reads context (mate_idx = -1, eq = [0, 1)) and the rescue pass and the final consensus update are off, so the sets differ
slightly from the batch run's; the distribution is an estimate of the run's, not a replay of it.

    python bench/hit_sizes.py [--pairs 1000000] [--streams 4096] [--sample 24] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from trust4_b200 import api, synth  # noqa: E402


def prefix_stats(h):
    """h: int32[n, 5] {seqIdx, seqOffset, readOffset, strand, repeats}.  Bits that vary in the key prefix, and the
    width of the field-wise rank the device sorts on (strand bit + contig range + diagonal range)."""
    s = (h[:, 3] == 1).astype(np.uint64)
    idx = h[:, 0].astype(np.uint64)
    c = (h[:, 2].astype(np.int64) - h[:, 1] + (1 << 20)).astype(np.uint64)
    p = (s << np.uint64(43)) | (idx << np.uint64(21)) | c
    vary = int(np.bitwise_or.reduce(p) ^ np.bitwise_and.reduce(p))
    rank_bits = int(s.min() != s.max()) + int(idx.max() - idx.min()).bit_length() + int(c.max() - c.min()).bit_length()
    return bin(vary).count("1"), vary.bit_length() - (vary & -vary).bit_length() + 1 if vary else 0, rank_bits


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--pairs", type=int, default=1000000)
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--sample", type=int, default=24, help="streams drawn uniformly")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    lib = api.default_lib()
    lib.check(lib.init(0, 0))
    cl = synth.make_clones(max(20, args.pairs // 50), args.seed)
    rd = synth.sample_pairs(cl, args.pairs, 150, args.seed * 1000)
    w = synth.build_workload(cl, rd, device=torch.device("cuda", 0))
    off, descs = synth.shard_workload(w, args.streams, group="gene")
    pool = np.ascontiguousarray(w.pool)
    cfg1 = synth.run_cfg(do_rescue=0, final_update=0)
    pick = np.random.default_rng(12345).permutation(len(off) - 1)[:args.sample]
    H, nset, span, rank = [], [], [], []
    for j in pick:
        lib.check(lib.reset())
        s = api.SeqSet(9, lib)
        for d in descs[off[j]:off[j + 1]]:
            if d["flags"] & 2:      # T4_RD_FILTERED: the driver skips it
                continue
            read = bytes(pool[int(d["seq_off"]):int(d["seq_off"]) + int(d["len"])]).decode()
            h = s.get_hits(read, int(d["strand_in"]), int(d["barcode"]), False)
            H.append(len(h))
            if len(h):
                a, b, c = prefix_stats(h)
                nset.append(a)
                span.append(b)
                rank.append(c)
            one = d.copy()
            one["mate_idx"], one["eq_lo"], one["eq_hi"] = -1, 0, 1
            s.run_descs(cfg1, np.array([one]), pool, w.names)
        s.close()
    H = np.array(H)
    q = lambda x, p: float(np.percentile(x, p)) if len(x) else None  # noqa: E731
    res = {"streams": int(len(pick)), "reads": int(len(H)),
           "hits": {"mean": float(H.mean()), "median": q(H, 50), "p90": q(H, 90), "p99": q(H, 99), "max": int(H.max()),
                    "frac_le_1024": float((H <= 1024).mean()), "frac_le_2048": float((H <= 2048).mean()),
                    "frac_le_4096": float((H <= 4096).mean())},
           "prefix_bits_varying": {"median": q(nset, 50), "p99": q(nset, 99)},
           "prefix_span_bits": {"median": q(span, 50), "p99": q(span, 99)},
           "rank_bits": {"median": q(rank, 50), "p99": q(rank, 99), "max": int(max(rank)) if rank else None}}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
