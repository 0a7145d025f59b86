#!/usr/bin/env python3
"""Per-cell 21-mer statistics and barcode sort of a --barcode run: the device against the reference's CPU loop.

    python bench/barcode_stats.py [--barcodes 1000] [--reads-per-barcode 2000] [--steps 5] [--warmup 2] [--threads N]

Input: configs[3]-shaped barcoded reads from trust4_b200.synth (the defaults are `bench.py --config 3`'s: 1000 cells x 2000
150 bp single-end reads).  It measures
  * device_count_stats_ms: t4_barcode_kmer_count_stats_device on buffers already on the GPU (count + statistics
    launches of every pass), CUDA events, median of --steps runs after --warmup;
  * device_sort_ms: t4_sort_reads_barcode (CompReadWithBarcode order), a host-buffer call: wall time, its own copies included;
  * h2d_ms / d2h_ms: the copies the count needs around the device form (reads, offsets, lengths, barcodes in; three
    statistics out), CUDA events;
  * ref_count_stats_ms: the reference's barcode-wise loop (KmerCount.hpp compiled into oracle/_ref/libt4ref.so, one
    t4ref_kmer_count_stats call per cell) on --threads host threads, barcodes dealt out by barcode % threads as
    BarcodeKmerCount_Thread does (main.cpp:569-604).  Each call builds a fresh KmerCount( 21 ) where the driver clears one
    KmerCount( 21, 23 ); ref_fresh_table_ms is what building one costs alone (ref_cells_per_thread of them run one after
    another on each thread), so the driver's own loop is faster than ref_count_stats_ms by up to about their product.
It checks the device's statistics for a seeded sample of cells and the sort order against the reference (std::sort under
_sortRead::operator< within each (barcode, barcodeMinCnt) group), and prints one JSON line with the card name and its
power limit read in the same run.  It writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(int(os.environ.get("LOCAL_RANK", 0))), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.split("\n")[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--barcodes", type=int, default=1000)
    ap.add_argument("--reads-per-barcode", type=int, default=2000)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1, help="host threads of the reference loop")
    ap.add_argument("--sample-cells", type=int, default=64, help="cells whose statistics are compared read by read")
    args = ap.parse_args()

    import torch
    from trust4_b200 import api, synth
    import refharness as rh
    import barcode_cases as bcc
    from parity_cases import _check_sorted_records

    lib = api.default_lib()
    lib.check(lib.init(0, 2 << 30))
    cl = synth.make_clones(max(20, 2 * args.barcodes), args.seed)
    rd, bc = synth.sample_single_cell(cl, args.barcodes, args.reads_per_barcode, 150, args.seed * 1000)
    n, L = rd.codes.shape
    pool = np.concatenate([np.frombuffer(b"ACGT", dtype=np.uint8)[rd.codes].reshape(-1), np.zeros(16, dtype=np.uint8)])
    off = np.arange(n, dtype=np.uint64) * np.uint64(L)
    lens = np.full(n, L, dtype=np.int32)
    bc = bc.astype(np.int32)
    tb = lib.kmer_count_table_bytes(int(n * (L - 20)))

    dev = torch.device("cuda", 0)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    host = [torch.from_numpy(a).pin_memory() for a in (pool, off.view(np.int64), lens, bc)]
    d_in = [torch.empty_like(h, device=dev) for h in host]
    table = torch.empty(tb, dtype=torch.uint8, device=dev)
    d_out = [torch.empty(n, dtype=t, device=dev) for t in (torch.int32, torch.int32, torch.float32)]
    h_out = [torch.empty(n, dtype=t).pin_memory() for t in (torch.int32, torch.int32, torch.float32)]
    stream = torch.cuda.current_stream().cuda_stream

    def count():
        lib.check(lib.barcode_kmer_count_stats_device(d_in[0].data_ptr(), d_in[1].data_ptr(), d_in[2].data_ptr(), d_in[3].data_ptr(), n,
                                                      int(bc.max()), 21, table.data_ptr(), tb, d_out[0].data_ptr(), d_out[1].data_ptr(),
                                                      d_out[2].data_ptr(), stream))

    h2d, d2h, dev_ms = [], [], []
    for it in range(args.warmup + args.steps):
        e = [ev() for _ in range(4)]
        e[0].record()
        for d, h in zip(d_in, host):
            d.copy_(h, non_blocking=True)
        e[1].record()
        count()
        e[2].record()
        for h, d in zip(h_out, d_out):
            h.copy_(d, non_blocking=True)
        e[3].record()
        torch.cuda.synchronize()
        st = np.zeros(4, dtype=np.uint64)
        lib.check(lib.kmer_count_table_stats(table.data_ptr(), tb, st.ctypes.data))
        assert st[3] == 0, "count table overflow"
        if it >= args.warmup:
            h2d.append(e[0].elapsed_time(e[1]))
            dev_ms.append(e[1].elapsed_time(e[2]))
            d2h.append(e[2].elapsed_time(e[3]))
    gmn, gmed, gavg = (h.numpy().copy() for h in h_out)

    # the reference's per-cell loop on --threads host threads, barcodes dealt out by barcode % threads
    # (BarcodeKmerCount_Thread); the input is grouped by barcode, as sample_single_cell returns it.  Each cell is one
    # t4ref_kmer_count_stats call (ctypes releases the GIL): a fresh KmerCount( 21 ) over the cell's reads, where the driver
    # reuses one KmerCount( 21, 23 ) with Clear().  The results are the same; the fresh object's 1 000 003 empty maps cost
    # time the driver does not spend, measured alone as ref_fresh_table_ms and reported next to the total.
    assert (np.diff(bc) >= 0).all()
    rmn, rmed = np.zeros(n, np.int32), np.zeros(n, np.int32)
    ravg, rnl = np.zeros(n, np.float32), np.zeros(n, np.int32)
    rl = rh.lib()
    groups = bcc.barcode_groups(bc)

    def ref_worker(t):
        for g in groups:
            if int(bc[g[0]]) % args.threads != t:
                continue
            i, m = int(g[0]), len(g)
            rl.t4ref_kmer_count_stats(pool.ctypes.data, None, off.ctypes.data + 8 * i, lens.ctypes.data + 4 * i, m, 21, rmn.ctypes.data + 4 * i,
                                      rmed.ctypes.data + 4 * i, ravg.ctypes.data + 4 * i, rnl.ctypes.data + 4 * i)

    t0 = time.perf_counter()
    th = [threading.Thread(target=ref_worker, args=(t,)) for t in range(args.threads)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    ref_ms = (time.perf_counter() - t0) * 1e3
    fresh = []
    for _ in range(5):
        t0 = time.perf_counter()
        rl.t4ref_kmer_count_stats(pool.ctypes.data, None, off.ctypes.data, lens.ctypes.data, 0, 21, rmn.ctypes.data, rmed.ctypes.data,
                                  ravg.ctypes.data, rnl.ctypes.data)
        fresh.append((time.perf_counter() - t0) * 1e3)
    rng = np.random.default_rng(args.seed)
    cells = rng.choice(args.barcodes, size=min(args.sample_cells, args.barcodes), replace=False)
    sel = np.isin(bc, cells)
    stats_equal = bool((gmn[sel] == rmn[sel]).all() and (gmed[sel] == rmed[sel]).all()
                       and (gavg[sel].view(np.uint32) == ravg[sel].view(np.uint32)).all())

    # the sort, with the per-cell statistics just computed; global statistics from the device's global count
    mn, med, avg, _ = api.kmer_count_stats(pool, off, lens, 21, lib)
    ids = [b"r%d" % i for i in range(n)]
    sort_ms = []
    for it in range(args.warmup + args.steps):
        t0 = time.perf_counter()
        go = api.sort_reads_barcode(pool, off, lens, ids, mn, med, avg, bc, gmn, lib)
        if it >= args.warmup:
            sort_ms.append((time.perf_counter() - t0) * 1e3)
    pb = pool.tobytes()
    reads = [pb[o:o + L] for o in off.tolist()]
    ro = bcc._ref_sort_bc(rh, reads, ids, mn, med, avg, bc, gmn)
    key = bcc.bc_key(reads, ids, mn.tolist(), med.tolist(), avg.tolist(), bc.tolist(), gmn.tolist())
    keys = [key(i) for i in range(n)]
    try:
        _check_sorted_records(go, keys, ro)
        sort_equal = True
    except AssertionError:
        sort_equal = False

    med_ms = statistics.median
    print(json.dumps({
        "bench": "barcode_stats", "card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
        "cells": args.barcodes, "reads_per_cell": args.reads_per_barcode, "reads": int(n), "read_len": int(L),
        "steps": args.steps, "warmup": args.warmup,
        "device_count_stats_ms": round(med_ms(dev_ms), 3), "h2d_ms": round(med_ms(h2d), 3), "d2h_ms": round(med_ms(d2h), 3),
        "device_sort_ms": round(med_ms(sort_ms), 3),
        "ref_count_stats_ms": round(ref_ms, 1), "ref_threads": args.threads,
        "ref_fresh_table_ms": round(med_ms(fresh), 2), "ref_cells_per_thread": -(-len(groups) // args.threads),
        "sample_cells": int(len(cells)), "stats_equal_reference": stats_equal, "sort_equal_reference": sort_equal,
    }))
    return 0 if stats_equal and sort_equal else 1


if __name__ == "__main__":
    sys.exit(main())
