#!/usr/bin/env python3
"""Generate the stage-0 drop-in driver: the reference FastqExtractor.cpp with its candidate test answered by the device.

    python make_extractor_main.py <reference FastqExtractor.cpp> <output .cpp>

Five places change; each is found by its exact text and must occur once (FastqExtractor.cpp line numbers):
  * `if ( threadCnt == 1 )` in front of the per-read loop (:492) becomes `if ( T4_EXTRACT_SERIAL( threadCnt ) )`, which is
    false: every -t runs the batched branch (:551-720), so every read goes through the device scan;
  * `int maxBatchSize = 512 * threadCnt ;` (:551) becomes `int maxBatchSize = T4_EXTRACT_BATCH_SIZE( threadCnt ) ;`
    (at least 2^18 reads; the output order is the input order whatever the batch size);
  * `T4_EXTRACT_SCAN() ;` goes in front of the loop that starts the worker threads (:627-631): one t4_refset_scan call over
    read 1 and, with mates, one over read 2 of the batch;
  * the two `IsGoodCandidate( arg.readBatch[2][i].seq, ... )` calls of ProcessReads_Thread (:209, :212) become
    `T4_EXTRACT_CANDIDATE( mate, i, ... )`: the answer the scan recorded for that batch slot stands in for the call;
  * `T4_EXTRACT_DONE() ;` goes in front of `PrintLog( "Finish extracting reads." )` (:731): the route line on stderr.
The macros are defined by t4_extractor_adapter.hpp (force-included); everything else of FastqExtractor.cpp is used as it
is.  The output is a build artefact (integration/_build/, git-ignored) -- no reference source is kept in this repository."""
import sys


def main():
    src, dst = sys.argv[1], sys.argv[2]
    lines = open(src).read().split("\n")

    def one(text, what):
        at = [i for i, l in enumerate(lines) if l == text]
        if len(at) != 1:
            sys.exit("make_extractor_main: %s (%r) not found exactly once" % (what, text))
        return at[0]

    def replace(i, old, new):
        if lines[i].count(old) != 1:
            sys.exit("make_extractor_main: %r not found once in line %d" % (old, i + 1))
        lines[i] = lines[i].replace(old, new)

    c1 = one("\t\tif ( IsGoodCandidate( arg.readBatch[i].seq, arg.buffer, arg.refSet ) )", "read 1's candidate test")
    c2 = one("\t\tif ( !goodCandidate && arg.readBatch2 && IsGoodCandidate( arg.readBatch2[i].seq, arg.buffer, arg.refSet ) )",
             "read 2's candidate test")
    serial = one("\tif ( threadCnt == 1 )", "the per-read branch")
    batch = one("\t\tint maxBatchSize = 512 * threadCnt ;", "the batch size")
    done = one('\tPrintLog( "Finish extracting reads." ) ;', "the last log line")
    start = [i for i, l in enumerate(lines) if l == "\t\t\tfor ( i = 0 ; i < threadCnt ; ++i )"
             and i + 3 < len(lines) and lines[i + 2].strip() == "args[i].batchSize = batchSize ;"
             and lines[i + 3].strip().startswith("pthread_create(")]
    if len(start) != 1 or not batch < start[0] < done:
        sys.exit("make_extractor_main: the loop that starts the worker threads of a batch was not found")
    start = start[0]
    if not c1 < c2 < serial < batch < start < done:
        sys.exit("make_extractor_main: the anchors are not in the expected order")

    replace(c1, "IsGoodCandidate( arg.readBatch[i].seq,", "T4_EXTRACT_CANDIDATE( 0, i, arg.readBatch[i].seq,")
    replace(c2, "IsGoodCandidate( arg.readBatch2[i].seq,", "T4_EXTRACT_CANDIDATE( 1, i, arg.readBatch2[i].seq,")
    replace(serial, "threadCnt == 1", "T4_EXTRACT_SERIAL( threadCnt )")
    replace(batch, "512 * threadCnt", "T4_EXTRACT_BATCH_SIZE( threadCnt )")
    out = (lines[:start] + ["\t\t\tT4_EXTRACT_SCAN() ; // trust4_b200 stage-0 route (integration/t4_extractor_adapter.hpp)",
                            '#line %d "%s"' % (start + 1, src)] + lines[start:done]
           + ["\tT4_EXTRACT_DONE() ; // trust4_b200 stage-0 route: the route line on stderr",
              '#line %d "%s"' % (done + 1, src)] + lines[done:])
    open(dst, "w").write('#line 1 "%s"\n' % src + "\n".join(out))
    print("make_extractor_main: candidate tests at lines %d and %d, per-read branch at line %d, batch size at line %d, "
          "T4_EXTRACT_SCAN() before line %d and T4_EXTRACT_DONE() before line %d of %s"
          % (c1 + 1, c2 + 1, serial + 1, batch + 1, start + 1, done + 1, src))


if __name__ == "__main__":
    main()
