#!/usr/bin/env python3
"""Generate the batch-route driver: the reference main.cpp with one inserted line per offloaded pass (six).

    python make_batch_main.py <reference main.cpp> <output .cpp>

The line `T4_BATCH_PREPARE() ;` goes directly in front of the stage-1 AddRead loop (main.cpp:1583, the first
`for ( i = 0 ; i < readCnt ; ++i )` after `int prevAddRet = -1 ;`).  The line `T4_BATCH_ASSIGN()` (an `if ( !... )` without
a body) goes directly in front of the AssignRead loop (main.cpp:2075, the `if ( threadCnt <= 1 ) ... else ...` statement
after `extendedSeq.SetNovelSeqSimilarity( 0.95 ) ;`), which becomes its fall-back branch; `T4_BATCH_ANNOTATE()` (opt-in at
run time, T4_ANNOTATE=1) likewise in front of the rough annotation loop (main.cpp:1084) and `T4_BATCH_KMERSTATS()` (opt-in,
T4_KMERSTATS=1) in front of the count-statistics loop (main.cpp:981), `T4_BATCH_SORT()` (opt-in, T4_SORT=1) in front of the
`std::sort( sortedReads ... )` statement (main.cpp:1078), `T4_BATCH_BARCODE_STATS()` (opt-in, T4_BCSTATS=1) in front of
the barcode-wise statistics block `if (hasBarcode) { ... }` after the rough annotation (main.cpp:1123).  The macros are defined by
t4_seqset_adapter.hpp (force-included); everything else of main.cpp is used as it is.  The output is a build artefact (integration/_build/,
git-ignored) -- no reference source is kept in this repository."""
import sys


def main():
    src, dst = sys.argv[1], sys.argv[2]
    lines = open(src).read().split("\n")
    start = [i for i, l in enumerate(lines) if l.strip() == "int prevAddRet = -1 ;"]
    if len(start) != 1:
        sys.exit("make_batch_main: anchor 'int prevAddRet = -1 ;' not found exactly once")
    loop = None
    for i in range(start[0], len(lines)):
        if lines[i] == "\tfor ( i = 0 ; i < readCnt ; ++i )":
            loop = i
            break
    if loop is None or loop - start[0] > 80:
        sys.exit("make_batch_main: the AddRead loop header was not found after the anchor")
    kb = [i for i, l in enumerate(lines) if l == "\tkmerCount.SetBuffer( maxReadLen ) ;"]
    if len(kb) != 1 or lines[kb[0] + 1] != "\tif (threadCnt == 1)":
        sys.exit("make_batch_main: the count-statistics loop (`if (threadCnt == 1)` after kmerCount.SetBuffer) was not found")
    kst = kb[0] + 1
    srt = [i for i, l in enumerate(lines) if l == "\tstd::sort( sortedReads.begin(), sortedReads.end() ) ;"]
    srt = [i for i in srt if i > kst]     # (a second occurrence further down sits inside a comment block of the reference)
    if not srt:
        sys.exit("make_batch_main: `std::sort( sortedReads.begin(), sortedReads.end() ) ;` was not found after the statistics loop")
    srt = srt[0]
    rad = [i for i, l in enumerate(lines) if l == "\t\trefSet.SetRadius(0) ;"]
    if len(rad) != 1 or lines[rad[0] + 1] != "\tif ( threadCnt <= 1 )":
        sys.exit("make_batch_main: the rough annotation loop (`if ( threadCnt <= 1 )` after refSet.SetRadius(0)) was not found")
    ann = rad[0] + 1
    sim = [i for i, l in enumerate(lines) if l.strip() == "extendedSeq.SetNovelSeqSimilarity( 0.95 ) ;"]
    if len(sim) != 1 or lines[sim[0] + 1] != "\tif ( threadCnt <= 1 )":
        sys.exit("make_batch_main: the AssignRead loop (`if ( threadCnt <= 1 )` after SetNovelSeqSimilarity( 0.95 )) was not found")
    asg = sim[0] + 1
    bcs = [i for i, l in enumerate(lines) if l == "\tif (hasBarcode)" and ann < i < loop and "CompReadWithBarcode" in lines[i + 3]]
    if len(bcs) != 1 or lines[bcs[0] + 1] != "\t{":
        sys.exit("make_batch_main: the barcode-wise statistics block (`if (hasBarcode)` sorting with CompReadWithBarcode after the "
                 "rough annotation) was not found")
    bcs = bcs[0]
    out = (lines[:kst] + ["\tT4_BATCH_KMERSTATS() // trust4_b200 batch route (opt-in): the statement below is the fall-back branch",
                          '#line %d "%s"' % (kst + 1, src)] + lines[kst:srt]
           + ["\tT4_BATCH_SORT() // trust4_b200 batch route (opt-in): the statement below is the fall-back",
              '#line %d "%s"' % (srt + 1, src)] + lines[srt:ann]
           + ["\tT4_BATCH_ANNOTATE() // trust4_b200 batch route (opt-in): the statement below is the fall-back branch",
              '#line %d "%s"' % (ann + 1, src)] + lines[ann:bcs]
           + ["\tT4_BATCH_BARCODE_STATS() // trust4_b200 batch route (opt-in): the statement below is the fall-back branch",
              '#line %d "%s"' % (bcs + 1, src)] + lines[bcs:loop]
           + ["\tT4_BATCH_PREPARE() ; // trust4_b200 batch route (integration/t4_seqset_adapter.hpp)",
              '#line %d "%s"' % (loop + 1, src)] + lines[loop:asg]
           + ["\tT4_BATCH_ASSIGN() // trust4_b200 batch route: the statement below is the fall-back branch",
              '#line %d "%s"' % (asg + 1, src)] + lines[asg:])
    open(dst, "w").write("\n".join(out))
    print("make_batch_main: inserted T4_BATCH_KMERSTATS() before line %d, T4_BATCH_SORT() before line %d, T4_BATCH_ANNOTATE() before line %d, "
          "T4_BATCH_BARCODE_STATS() before line %d, T4_BATCH_PREPARE() before line %d and T4_BATCH_ASSIGN() before line %d of %s"
          % (kst + 1, srt + 1, ann + 1, bcs + 1, loop + 1, asg + 1, src))


if __name__ == "__main__":
    main()
