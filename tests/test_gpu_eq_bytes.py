"""The equality byte the engine keeps beside every posWeight column (one per column, bit b = IsBaseEqual( column, base b ),
read by the overhang masks, the gap scoring and the overhang DPs instead of the four counts) agrees with the counts after
every kind of posWeight update: new contigs, the commit, extension left and right (past capacity too), merges,
RepeatAddRead runs, a k change, barcode release, InputNovelFa, InputRefFa, reads of 201-512 bp and the AssignRead pass's
PREP copy and RECOMPUTE.  Each case also passes its own parity checks against the reference.  The emulation twins run the same cases on
the host build of the engine (tests/emu), which keeps the same bytes."""
import numpy as np
import pytest

import long_read_cases as lr
import parity_cases as pc
from trust4_b200 import api, synth


class _Sets:
    """Every set a case creates (since its last reset), so that their bytes can be checked once the case is done; the
    AssignRead pass's extended sets are checked just before the pass is freed."""

    def __init__(self, monkeypatch, lib):
        self.sets, self.cols, self.ext = [], 0, 0
        init, reset, close = api.SeqSet.__init__, lib.reset, api.Assign.close
        rec = self

        def seqset_init(s, *a, **kw):
            init(s, *a, **kw)
            if type(s) is api.SeqSet:      # borrowed sets belong to (and die with) their owner
                rec.sets.append(s)

        def lib_reset():
            rec.sets.clear()
            return reset()

        def assign_close(a):
            if a.h:
                for j in range(a.n_sets):
                    rec.ext += rec.check_one(a.extended_set(j))
            close(a)

        monkeypatch.setattr(api.SeqSet, "__init__", seqset_init)
        monkeypatch.setattr(lib, "reset", lib_reset)
        monkeypatch.setattr(api.Assign, "close", assign_close)

    @staticmethod
    def check_one(s):
        n, bad = s.check_eq_bytes()
        assert bad == 0, ("equality bytes disagree with posWeight", bad, n)
        return n

    def check(self):
        """Columns checked over the live sets (every byte must agree)."""
        self.cols += sum(self.check_one(s) for s in self.sets if s.h)
        return self.cols


def _change_k(lib, ref):
    lib.check(lib.reset())
    w = pc.small_workload(21, 60, 1500)
    cfg = synth.run_cfg(change_k_threshold=20)     # k: 9 -> 11 -> 13 early
    g = api.SeqSet(9, lib)
    r = ref.RefSeqSet(9)
    _, gret, _, _ = g.run_descs(cfg, w.descs, w.pool, w.names)
    _, rret, _, _ = r.run_descs(cfg, w.descs, w.pool, w.names)
    assert g.kmer_length() == r.kmer_length() > 9
    assert (gret == rret).all() and g.output() == r.output()


def _ref_set(lib, tmp):
    """InputRefFa: the reference gene set's contigs (all counts zero) are checked before the set is freed."""
    lib.check(lib.reset())
    fa = str(tmp / "genes.fa")
    pc.write_gene_fasta(fa)
    rs = api.RefSet(fa, 9, lib)
    n = _Sets.check_one(rs.seqset())
    rs.close()
    assert n > 0


def _repeat_last(lib, ref):
    """A RepeatAddRead run as the contig's last update, turning a mixed column (one count of each of two bases, both
    bits set) into a one-base column: the bytes are only right if RepeatAddRead refreshed them."""
    lib.check(lib.reset())
    rng = np.random.default_rng(5)
    x = "".join("ACGT"[c] for c in rng.integers(0, 4, size=150))
    y = x[:75] + "ACGT".replace(x[75], "")[0] + x[76:]
    g, r = api.SeqSet(9, lib), ref.RefSeqSet(9)
    for s in (g, r):
        s.input_novel_read("IGHV1-2*01", x, 1, -1)
        assert s.add_read(y, "IGHV", 0, -1, 1, 0, 0.9)[0] == 0
        for _ in range(3):
            s.repeat_add_read(y)
    assert g.output() == r.output()


def _size(emu):
    return dict(nclones=25, npairs=400) if emu else dict(nclones=40, npairs=1500)


CASES = {
    # workloads with stored reference results (tests/golden/batch_ref.json.gz)
    "batch_s1": lambda lib, ref, tmp, emu: pc.check_batch_vs_ref(lib, ref, 1, 1, **_size(emu)),
    "batch_s3": lambda lib, ref, tmp, emu: pc.check_batch_vs_ref(lib, ref, 2, 3, **_size(emu)),
    "gene_streams": lambda lib, ref, tmp, emu: pc.check_batch_vs_ref(lib, ref, 8, 9, nclones=40, npairs=700, group="gene"),
    "growth_and_merges": lambda lib, ref, tmp, emu: pc.check_batch_vs_ref(lib, ref, 9, 1, nclones=300, npairs=6000),
    "growth_past_capacity": lambda lib, ref, tmp, emu: lr.check_contig_growth(lib, ref),
    "repeat_add_last": lambda lib, ref, tmp, emu: _repeat_last(lib, ref),
    "duplicate_runs": lambda lib, ref, tmp, emu: pc.check_dup_runs(lib, ref),
    "k_change": lambda lib, ref, tmp, emu: _change_k(lib, ref),
    "barcode_release": lambda lib, ref, tmp, emu: pc.check_barcode_release(lib, ref),
    "input_novel_fa": lambda lib, ref, tmp, emu: pc.check_input_novel_fa(lib, ref, tmp),
    "long_reads_gaps": lambda lib, ref, tmp, emu: lr.check_gap_scoring(lib, ref, 9),
    "long_reads_sides": lambda lib, ref, tmp, emu: lr.check_extend_sides(lib, ref, 20),
    "ref_input_fa": lambda lib, ref, tmp, emu: _ref_set(lib, tmp),
    "assign_recompute": lambda lib, ref, tmp, emu: pc.check_assign_pass(lib, ref, 81, 3, nclones=30 if emu else 60,
                                                                         npairs=500 if emu else 2500),
}


def _run(case, lib, ref, tmp_path, monkeypatch, emu):
    rec = _Sets(monkeypatch, lib)
    CASES[case](lib, ref, tmp_path, emu)
    assert rec.check() > 0 or case == "ref_input_fa"
    if case == "assign_recompute":
        assert rec.ext > 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_gpu_eq_bytes_follow_posweight(gpu_lib, ref, tmp_path, monkeypatch, case):
    _run(case, gpu_lib, ref, tmp_path, monkeypatch, emu=False)


@pytest.mark.parametrize("case", list(CASES))
def test_emu_eq_bytes_follow_posweight(emu_lib, ref, tmp_path, monkeypatch, case):
    _run(case, emu_lib, ref, tmp_path, monkeypatch, emu=True)
