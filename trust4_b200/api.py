"""ctypes mirror of include/trust4_b200.h (host side, Python).

`SeqSet` mirrors the reference class of the same name for the stage-1 path
(SeqSet.hpp: AddRead :3426, RepeatAddRead :4477, InputNovelRead :3028,
UpdateAllConsensus :4525, ChangeKmerLength :4624, Output :10939) with the same
argument meaning and return codes; everything executes on the GPU through
libtrust4_b200.so.  There is no CPU fallback: loading fails loudly when the
extension is missing, and every call fails with T4_E_NODEVICE without a GPU.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("T4_LIB_PATH") or os.path.join(_HERE, "libtrust4_b200.so")     # T4_LIB_PATH: build variants for experiments

T4_E_BASE = -16
T4_E_CUDA, T4_E_NOMEM, T4_E_INVAL, T4_E_UNSUPPORTED, T4_E_NODEVICE, T4_E_INTERNAL = -17, -18, -19, -20, -21, -22
N_COUNTERS = 24

EXPORTS = [
    "init", "shutdown", "last_error", "version", "arena_stats", "reset",
    "seqset_create", "seqsets_create", "seqsets_create_ex", "seqset_destroy", "seqset_set_hit_len_required",
    "seqset_set_novel_seq_similarity", "seqset_set_consider_barcode_in_hash", "seqset_set_is_long",
    "seqset_size", "seqset_kmer_length", "seqset_add_read", "seqset_repeat_add_read",
    "seqset_input_novel_read", "seqset_update_all_consensus", "seqset_change_kmer_length",
    "seqset_output", "seqset_output_mem", "free", "seqset_get_contig", "has_motif",
    "reverse_complement_in_place", "seqset_get_hits", "seqset_get_overlaps", "dp_pos_weight_batch", "dp_hot_path_batch",
    "seqset_add_reads_batch", "streams_run", "workload_upload", "workload_free",
    "streams_run_resident", "workload_results", "workload_events", "shard_reads", "last_counters", "stream_residency", "streams_error",
    "hits_create", "hits_free", "streams_get_hits", "hits_stats", "hits_fetch", "hits_device_buffers",
    "seqset_index_checksum", "streams_pack_contigs", "streams_cycles",
    "seqset_release_finished_barcode", "seqset_release_shallow_contigs", "seqset_input_novel_fa", "seqset_contig_flags",
    "streams_assign_reads", "assign_free", "assign_results", "assign_stats", "assign_extended_set", "assign_device_buffers",
    "kmer_count_stats", "kmer_count_table_bytes", "kmer_count_stats_device", "kmer_count_table_stats",
    "refset_create_from_fa", "refset_free", "refset_size", "refset_name", "refset_seqset", "refset_set_hit_len_required",
    "refset_set_radius", "refset_scan", "refset_scan_device", "test_lis", "test_check_eq_bytes", "test_group_hits", "refset_get_overlaps", "refset_annotate", "sort_reads", "mate_overlap_batch",
    "barcode_kmer_count_stats", "barcode_kmer_count_stats_device", "sort_reads_barcode",
]


class T4Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("trust4_b200 error %d: %s" % (code, msg))
        self.code = code


class Lib:
    """One loaded C-ABI library.  prefix is 't4_' for the product and 't4emu_' for the test emulation."""

    def __init__(self, path=LIB_PATH, prefix="t4_"):
        if not os.path.exists(path):
            raise ImportError(
                "%s not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'). "
                "trust4_b200 has no CPU fallback." % path)
        self.path = path
        self.prefix = prefix
        self.dll = C.CDLL(path)
        f = self._f
        vp, ci, cd, cs = C.c_void_p, C.c_int, C.c_double, C.c_char_p
        f("init", ci, [ci, C.c_size_t])
        f("shutdown", ci, [])
        f("reset", ci, [])
        f("last_error", cs, [])
        f("version", cs, [])
        f("arena_stats", ci, [C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)])
        f("seqset_create", vp, [ci])
        f("seqsets_create", ci, [ci, ci, C.POINTER(vp)])
        f("seqsets_create_ex", ci, [ci, ci, ci, ci, C.POINTER(vp)])
        f("seqset_destroy", None, [vp])
        f("seqset_set_hit_len_required", ci, [vp, ci])
        f("seqset_set_novel_seq_similarity", ci, [vp, cd])
        f("seqset_set_consider_barcode_in_hash", ci, [vp, ci])
        f("seqset_set_is_long", ci, [vp, ci])
        f("seqset_size", ci, [vp])
        f("seqset_kmer_length", ci, [vp])
        f("seqset_add_read", ci, [vp, cs, cs, C.POINTER(ci), ci, ci, ci, cd])
        f("seqset_repeat_add_read", ci, [vp, cs])
        f("seqset_input_novel_read", ci, [vp, cs, cs, ci, ci])
        f("seqset_update_all_consensus", ci, [vp])
        f("seqset_change_kmer_length", ci, [vp, ci])
        f("seqset_output_mem", ci, [vp, C.POINTER(vp), C.POINTER(C.c_size_t)])
        f("free", None, [vp])
        f("seqset_get_contig", ci, [vp, ci, cs, ci, vp, cs, ci, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), C.POINTER(ci)])
        f("has_motif", ci, [cs, ci])
        f("reverse_complement_in_place", None, [cs, ci])
        f("seqset_get_hits", ci, [vp, cs, ci, ci, ci, vp, ci])
        f("seqset_get_overlaps", ci, [vp, cs, ci, ci, ci, vp, vp, ci])
        f("dp_pos_weight_batch", ci, [ci, vp, vp, vp, vp, vp, vp, vp])
        f("dp_hot_path_batch", ci, [ci, ci, vp, vp, vp, vp, vp, vp])
        f("seqset_release_finished_barcode", ci, [vp, ci, ci])
        f("seqset_release_shallow_contigs", ci, [vp, ci])
        f("seqset_input_novel_fa", ci, [vp, cs])
        f("seqset_contig_flags", ci, [vp, ci])
        f("seqset_add_reads_batch", ci, [vp, vp, vp, ci, vp, C.c_size_t, C.POINTER(cs), ci, vp, vp, vp])
        f("streams_run", ci, [C.POINTER(vp), ci, vp, vp, vp, vp, C.c_size_t, C.POINTER(cs), ci, vp, vp, vp])
        f("workload_upload", vp, [vp, C.c_int64, vp, C.c_size_t, C.POINTER(cs), ci])
        f("workload_free", None, [vp])
        f("streams_run_resident", ci, [C.POINTER(vp), ci, vp, vp, vp, vp])
        f("workload_results", ci, [vp, vp, vp, vp])
        f("workload_events", ci, [vp, vp])
        f("shard_reads", ci, [vp, C.c_int64, ci, ci, vp, vp])
        f("last_counters", ci, [vp])
        f("stream_residency", ci, [C.POINTER(ci), C.POINTER(ci)])
        f("hits_create", vp, [C.c_int64, C.c_size_t])
        f("hits_free", None, [vp])
        f("streams_get_hits", ci, [C.POINTER(vp), ci, vp, vp, ci, vp, vp])
        f("hits_stats", ci, [vp, vp])
        f("hits_fetch", ci, [vp, C.c_int64, vp, ci, C.POINTER(ci)])
        f("hits_device_buffers", ci, [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)])
        f("streams_error", ci, [C.POINTER(vp), ci])
        f("seqset_index_checksum", C.c_int64, [vp, C.POINTER(C.c_uint64)])
        f("streams_cycles", ci, [C.POINTER(vp), ci, vp])
        f("streams_pack_contigs", ci, [C.POINTER(vp), ci, vp, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int64)])
        f("streams_assign_reads", vp, [C.POINTER(vp), ci, vp, vp, ci, ci, vp])
        f("assign_free", None, [vp])
        f("assign_results", ci, [vp, vp, vp])
        f("assign_stats", ci, [vp, vp])
        f("assign_extended_set", vp, [vp, ci])
        f("assign_device_buffers", ci, [vp, C.POINTER(vp), C.POINTER(vp)])
        f("kmer_count_stats", ci, [vp, vp, C.c_size_t, vp, vp, C.c_int64, ci, vp, vp, vp, vp])
        f("kmer_count_table_bytes", C.c_size_t, [C.c_int64])
        f("kmer_count_stats_device", ci, [vp, vp, vp, vp, C.c_int64, ci, vp, C.c_size_t, vp, vp, vp, vp, vp])
        f("kmer_count_table_stats", ci, [vp, C.c_size_t, vp])
        f("refset_create_from_fa", vp, [cs, ci])
        f("refset_free", None, [vp])
        f("refset_size", ci, [vp])
        f("refset_name", cs, [vp, ci])
        f("refset_seqset", vp, [vp])
        f("refset_set_hit_len_required", ci, [vp, ci])
        f("refset_set_radius", ci, [vp, ci])
        f("refset_scan", ci, [vp, vp, C.c_size_t, vp, vp, C.c_int64, vp, vp, vp])
        f("refset_scan_device", ci, [vp, vp, vp, vp, C.c_int64, vp, vp, vp, ci, vp])
        f("test_lis", ci, [vp, vp, ci, vp, vp])
        f("refset_get_overlaps", ci, [vp, cs, vp, vp, ci])
        f("refset_annotate", ci, [vp, vp, C.c_size_t, vp, vp, C.c_int64, vp, vp])
        f("sort_reads", ci, [vp, C.c_size_t, vp, vp, vp, C.c_size_t, vp, vp, vp, vp, C.c_int64, vp])
        f("mate_overlap_batch", ci, [vp, C.c_size_t, vp, vp, vp, vp, vp, vp, C.c_int64, vp, vp, vp])
        f("barcode_kmer_count_stats", ci, [vp, C.c_size_t, vp, vp, vp, C.c_int64, ci, vp, vp, vp])
        f("barcode_kmer_count_stats_device", ci, [vp, vp, vp, vp, C.c_int64, C.c_int32, ci, vp, C.c_size_t, vp, vp, vp, vp])
        f("sort_reads_barcode", ci, [vp, C.c_size_t, vp, vp, vp, C.c_size_t, vp, vp, vp, vp, vp, vp, C.c_int64, vp])

    def _f(self, name, restype, argtypes):
        fn = getattr(self.dll, self.prefix + name)
        fn.restype = restype
        fn.argtypes = argtypes
        setattr(self, name, fn)

    def err(self):
        return (self.last_error() or b"").decode()

    def check(self, r):
        if r < T4_E_BASE:
            raise T4Error(r, self.err())
        return r


_default = None


def default_lib() -> Lib:
    global _default
    if _default is None:
        _default = Lib()
    return _default


def _names_array(names):
    arr = (C.c_char_p * max(1, len(names)))(*[n if isinstance(n, bytes) else n.encode() for n in names])
    return arr


class SeqSet:
    """GPU-resident novel-contig set; method names follow the reference's SeqSet."""

    def __init__(self, k=9, lib: Lib | None = None, handle=None):
        self.lib = lib or default_lib()
        if handle is None:
            handle = self.lib.seqset_create(k)
            if not handle:
                raise T4Error(T4_E_CUDA, self.lib.err())
        self.h = C.c_void_p(handle)

    @classmethod
    def create_many(cls, n, k=9, lib: Lib | None = None, hit_len_required=31, consider_barcode=0):
        lib = lib or default_lib()
        arr = (C.c_void_p * n)()
        lib.check(lib.seqsets_create_ex(n, k, hit_len_required, consider_barcode, arr))
        return [cls(k, lib, arr[i]) for i in range(n)]

    def close(self):
        if self.h:
            self.lib.seqset_destroy(self.h)
            self.h = None

    def set_hit_len_required(self, v):
        return self.lib.check(self.lib.seqset_set_hit_len_required(self.h, v))

    def set_novel_seq_similarity(self, v):
        return self.lib.check(self.lib.seqset_set_novel_seq_similarity(self.h, v))

    def set_consider_barcode_in_hash(self, on):
        return self.lib.check(self.lib.seqset_set_consider_barcode_in_hash(self.h, int(on)))

    def set_is_long(self, on):
        return self.lib.check(self.lib.seqset_set_is_long(self.h, int(on)))

    def size(self):
        return self.lib.check(self.lib.seqset_size(self.h))

    def kmer_length(self):
        return self.lib.check(self.lib.seqset_kmer_length(self.h))

    def add_read(self, read, name, strand, barcode, min_kmer_count, repetitive, thr):
        s = C.c_int(strand)
        r = self.lib.seqset_add_read(self.h, read.encode(), name.encode(), C.byref(s), barcode, min_kmer_count, int(repetitive), thr)
        self.lib.check(r)
        return r, s.value

    def repeat_add_read(self, read):
        return self.lib.check(self.lib.seqset_repeat_add_read(self.h, read.encode()))

    def input_novel_read(self, name, read, strand, barcode):
        return self.lib.check(self.lib.seqset_input_novel_read(self.h, name.encode(), read.encode(), strand, barcode))

    def update_all_consensus(self):
        self.lib.check(self.lib.seqset_update_all_consensus(self.h))

    def change_kmer_length(self, k):
        self.lib.check(self.lib.seqset_change_kmer_length(self.h, k))

    def release_finished_barcode(self, barcode, contig_min_cov=0):
        """SeqSet::ReleaseFinishedBarcodeSeq({barcode}, true, contig_min_cov, true), SeqSet.hpp:10815."""
        self.lib.check(self.lib.seqset_release_finished_barcode(self.h, barcode, contig_min_cov))

    def release_shallow_contigs(self, min_cov):
        """SeqSet::ReleaseShallowContigs, SeqSet.hpp:10928."""
        self.lib.check(self.lib.seqset_release_shallow_contigs(self.h, min_cov))

    def input_novel_fa(self, filename):
        """SeqSet::InputNovelFa, SeqSet.hpp:2986."""
        return self.lib.check(self.lib.seqset_input_novel_fa(self.h, filename.encode()))

    def contig_flags(self, slot):
        return self.lib.seqset_contig_flags(self.h, slot)

    def output(self) -> bytes:
        buf = C.c_void_p()
        n = C.c_size_t()
        self.lib.check(self.lib.seqset_output_mem(self.h, C.byref(buf), C.byref(n)))
        s = C.string_at(buf, n.value)
        self.lib.free(buf)
        return s

    def get_hits(self, read, strand=0, barcode=-1, allow_total_skip=False, cap=1 << 20):
        out = np.zeros((cap, 5), dtype=np.int32)
        n = self.lib.check(self.lib.seqset_get_hits(self.h, read.encode(), strand, barcode, int(allow_total_skip), out.ctypes.data, cap))
        assert n <= cap
        return out[:n]

    def get_overlaps(self, read, strand=0, barcode=-1, skip_repeats=False, cap=1 << 14):
        out = np.zeros((cap, 8), dtype=np.int32)
        sim = np.zeros(cap, dtype=np.float64)
        n = self.lib.check(self.lib.seqset_get_overlaps(self.h, read.encode(), strand, barcode, int(skip_repeats), out.ctypes.data, sim.ctypes.data, cap))
        if n < 0:
            return n, None, None
        return n, out[:n], sim[:n]

    def check_eq_bytes(self):
        """(columns checked, columns whose equality byte disagrees with their posWeight counts) over every live contig."""
        if not hasattr(self.lib, "test_check_eq_bytes"):
            # resolved on first use, so that a build from before the cache (bench/ab_compare.py's parent) still loads
            self.lib._f("test_check_eq_bytes", C.c_int64, [C.c_void_p, C.POINTER(C.c_int64)])
        bad = C.c_int64(0)
        n = self.lib.test_check_eq_bytes(self.h, C.byref(bad))
        if n < 0:
            self.lib.check(int(n))
        return int(n), int(bad.value)

    def group_hits(self, keys):
        """t4_test_group_hits: the device's main hit sort and head pass over 64-bit hit keys in emission order.
        Returns (sorted keys, group heads, run heads), the heads over the valid keys and ending with their count."""
        if not hasattr(self.lib, "test_group_hits"):
            # resolved on first use, like check_eq_bytes
            self.lib._f("test_group_hits", C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p])
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        n = len(keys)
        out = np.zeros(max(n, 1), np.uint64)
        heads = np.zeros(2 * n + 4, np.int32)
        r = self.lib.check(self.lib.test_group_hits(self.h, keys.ctypes.data, n, out.ctypes.data, heads.ctypes.data))
        assert r == n
        nG, nR = int(heads[0]), int(heads[1])
        return out[:n], heads[2:3 + nG].astype(np.int64), heads[3 + nG:4 + nG + nR].astype(np.int64)

    def index_checksum(self):
        cs = C.c_uint64()
        n = self.lib.seqset_index_checksum(self.h, C.byref(cs))
        self.lib.check(int(n))
        return int(n), cs.value

    def get_contig(self, slot):
        ln = self.lib.seqset_get_contig(self.h, slot, None, 0, None, None, 0, None, None, None, None)
        if ln < 0:
            return None
        cons = C.create_string_buffer(ln + 1)
        pw = np.zeros((ln, 4), dtype=np.int32)
        name = C.create_string_buffer(4096)
        bc, nr, ml, mr = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        self.lib.seqset_get_contig(self.h, slot, cons, ln + 1, pw.ctypes.data, name, 4096, C.byref(bc), C.byref(nr), C.byref(ml), C.byref(mr))
        return dict(consensus=cons.value.decode(), pos_weight=pw, name=name.value.decode(), barcode=bc.value,
                    num_read=nr.value, min_left=ml.value, min_right=mr.value)

    def run_descs(self, cfg, descs, pool, names):
        """t4_seqset_add_reads_batch: the reference's AddRead loop over read descriptors."""
        n = len(descs)
        ret = np.zeros(n, dtype=np.int32)
        strands = np.zeros(n, dtype=np.int8)
        resc = np.zeros(n, dtype=np.int32)
        descs = np.ascontiguousarray(descs)
        pool = np.ascontiguousarray(pool)
        r = self.lib.seqset_add_reads_batch(self.h, cfg.ctypes.data, descs.ctypes.data, n, pool.ctypes.data, pool.nbytes,
                                            _names_array(names), len(names), ret.ctypes.data, strands.ctypes.data, resc.ctypes.data)
        self.lib.check(r)
        return int((ret >= 0).sum()), ret, strands, resc


def streams_run(sets, cfg, descs, desc_off, pool, names, lib: Lib | None = None):
    """t4_streams_run: one CTA per seqset, host buffers in and out."""
    lib = lib or sets[0].lib
    n = len(descs)
    ret = np.zeros(n, dtype=np.int32)
    strands = np.zeros(n, dtype=np.int8)
    resc = np.zeros(n, dtype=np.int32)
    descs = np.ascontiguousarray(descs)
    pool = np.ascontiguousarray(pool)
    desc_off = np.ascontiguousarray(desc_off, dtype=np.int64)
    hs = (C.c_void_p * len(sets))(*[s.h for s in sets])
    r = lib.streams_run(hs, len(sets), cfg.ctypes.data, descs.ctypes.data, desc_off.ctypes.data, pool.ctypes.data, pool.nbytes,
                        _names_array(names), len(names), ret.ctypes.data, strands.ctypes.data, resc.ctypes.data)
    lib.check(r)
    return ret, strands, resc


def dp_pos_weight_batch(problems, lib: Lib | None = None):
    """problems: list of (int32[lent,4], str).  Returns [(score, [edit ops])]."""
    lib = lib or default_lib()
    n = len(problems)
    t_off = np.zeros(n + 1, dtype=np.int64)
    p_off = np.zeros(n + 1, dtype=np.int64)
    a_off = np.zeros(n + 1, dtype=np.int64)
    for i, (tw, p) in enumerate(problems):
        t_off[i + 1] = t_off[i] + len(tw)
        p_off[i + 1] = p_off[i] + len(p)
        a_off[i + 1] = a_off[i] + len(tw) + len(p) + 2
    tw_all = np.zeros((max(1, t_off[n]), 4), dtype=np.int32)
    for i, (tw, p) in enumerate(problems):
        if len(tw):
            tw_all[t_off[i]:t_off[i + 1]] = tw
    p_all = np.frombuffer(("".join(p for _, p in problems) + "\0").encode(), dtype=np.uint8).copy()
    align = np.zeros(a_off[n] + 16, dtype=np.int8)
    score = np.zeros(n, dtype=np.int32)
    lib.check(lib.dp_pos_weight_batch(n, tw_all.ctypes.data, t_off.ctypes.data, p_all.ctypes.data, p_off.ctypes.data,
                                      align.ctypes.data, a_off.ctypes.data, score.ctypes.data))
    out = []
    for i in range(n):
        e = []
        for v in align[a_off[i]:a_off[i + 1]]:
            if v == -1:
                break
            e.append(int(v))
        out.append((int(score[i]), e))
    return out


def dp_hot_path_batch(problems, variant, lib: Lib | None = None):
    """Equal-length problems through the hot-path DP routines (t4_dp_hot_path_batch).  Returns [(score, [edit ops])];
    variant 2 (problems 2k, 2k+1 = a left and a right overhang side on one warp) returns [(matches, mismatches, indels, good)]."""
    lib = lib or default_lib()
    n = len(problems)
    off = np.zeros(n + 1, dtype=np.int64)
    a_off = np.zeros(n + 1, dtype=np.int64)
    for i, (tw, p) in enumerate(problems):
        assert len(tw) == len(p)
        off[i + 1] = off[i] + len(p)
        a_off[i + 1] = a_off[i] + ((max(2 * len(p) + 2, 16) + 3) & ~3)
    tw_all = np.zeros((max(1, off[n]), 4), dtype=np.int32)
    for i, (tw, p) in enumerate(problems):
        tw_all[off[i]:off[i + 1]] = tw
    p_all = np.frombuffer(("".join(p for _, p in problems) + "\0").encode(), dtype=np.uint8).copy()
    align = np.zeros(a_off[n] + 16, dtype=np.int8)
    score = np.zeros(n, dtype=np.int32)
    lib.check(lib.dp_hot_path_batch(n, variant, tw_all.ctypes.data, off.ctypes.data, p_all.ctypes.data,
                                    align.ctypes.data, a_off.ctypes.data, score.ctypes.data))
    if variant == 2:
        return [tuple(int(v) for v in align[a_off[i]:a_off[i] + 16].view(np.int32)) for i in range(n)]
    out = []
    for i in range(n):
        e = []
        for v in align[a_off[i]:a_off[i + 1]]:
            if v == -1:
                break
            e.append(int(v))
        out.append((int(score[i]), e))
    return out


class Workload:
    """Device-resident copy of a record list + read pool (t4_workload_upload); reads are 2-bit packed on upload."""

    def __init__(self, descs, pool, names, lib: Lib | None = None):
        self.lib = lib or default_lib()
        self.descs = np.ascontiguousarray(descs)
        self.pool = np.ascontiguousarray(pool)
        self.n = len(self.descs)
        self.h = self.lib.workload_upload(self.descs.ctypes.data, self.n, self.pool.ctypes.data, self.pool.nbytes,
                                          _names_array(names), len(names))
        if not self.h:
            raise T4Error(T4_E_NOMEM, self.lib.err())

    def close(self):
        if self.h:
            self.lib.workload_free(self.h)
            self.h = None


class Hits:
    """Result buffers of t4_streams_get_hits (device resident)."""

    def __init__(self, max_records, max_hits, lib: Lib | None = None):
        self.lib = lib or default_lib()
        self.h = self.lib.hits_create(max_records, max_hits)
        if not self.h:
            raise T4Error(T4_E_NOMEM, self.lib.err())

    def close(self):
        if self.h:
            self.lib.hits_free(self.h)
            self.h = None

    def stats(self):
        s = np.zeros(8, dtype=np.uint64)
        self.lib.check(self.lib.hits_stats(self.h, s.ctypes.data))
        return dict(hits=int(s[0]), lookups=int(s[1]), postings=int(s[2]), read_bytes=int(s[3]), algorithmic_bytes=int(s[4]),
                    algorithmic_bytes_16B_hits=int(s[5]), unsupported=int(s[6]), records=int(s[7]))

    def fetch(self, record, cap=1 << 16):
        out = np.zeros((cap, 4), dtype=np.int32)
        fl = C.c_int()
        n = self.lib.check(self.lib.hits_fetch(self.h, record, out.ctypes.data, cap, C.byref(fl)))
        if n > cap:
            return self.fetch(record, n)
        return out[:n], fl.value


def streams_get_hits(sets, wl: Workload, desc_off, hits: Hits, allow_total_skip=0, cuda_stream=None):
    """t4_streams_get_hits: SeqSet::GetHitsFromRead of every record against the (frozen) set of its stream."""
    lib = wl.lib
    off = np.ascontiguousarray(desc_off, dtype=np.int64)
    hs = (C.c_void_p * len(sets))(*[s.h if isinstance(s, SeqSet) else s for s in sets])
    lib.check(lib.streams_get_hits(hs, len(sets), wl.h, off.ctypes.data, int(allow_total_skip), cuda_stream, hits.h))


def kmer_count_stats(pool, seq_off, lens, k=21, lib: Lib | None = None, qual=None):
    """t4_kmer_count_stats: (min, median, avg, new_len) of the canonical k-mer counts of every read, counts taken over all
    the reads (KmerCount::AddCount + GetCountStatsAndTrim; qual = None: without the quality trimming)."""
    lib = lib or default_lib()
    pool = np.ascontiguousarray(pool)
    seq_off = np.ascontiguousarray(seq_off, dtype=np.uint64)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    n = len(lens)
    mn = np.zeros(max(1, n), dtype=np.int32)
    med = np.zeros(max(1, n), dtype=np.int32)
    avg = np.zeros(max(1, n), dtype=np.float32)
    nl = np.zeros(max(1, n), dtype=np.int32)
    if qual is not None:
        qual = np.ascontiguousarray(qual)
        assert qual.nbytes == pool.nbytes
    lib.check(lib.kmer_count_stats(pool.ctypes.data, qual.ctypes.data if qual is not None else None, pool.nbytes, seq_off.ctypes.data,
                                   lens.ctypes.data, n, int(k), mn.ctypes.data, med.ctypes.data, avg.ctypes.data, nl.ctypes.data))
    return mn[:n], med[:n], avg[:n], nl[:n]


def barcode_kmer_count_stats(pool, seq_off, lens, barcode, k=21, lib: Lib | None = None):
    """t4_barcode_kmer_count_stats: (barcodeMinCnt, barcodeMedianCnt, barcodeAvgCnt) of every read, its k-mers counted
    over the reads of its own barcode only (main.cpp:1128-1180).  Reads in any order; barcodes in [0, 2^31)."""
    lib = lib or default_lib()
    pool = np.ascontiguousarray(pool)
    seq_off = np.ascontiguousarray(seq_off, dtype=np.uint64)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    barcode = np.ascontiguousarray(barcode, dtype=np.int32)
    n = len(lens)
    assert len(barcode) == n
    mn = np.zeros(max(1, n), dtype=np.int32)
    med = np.zeros(max(1, n), dtype=np.int32)
    avg = np.zeros(max(1, n), dtype=np.float32)
    lib.check(lib.barcode_kmer_count_stats(pool.ctypes.data, pool.nbytes, seq_off.ctypes.data, lens.ctypes.data, barcode.ctypes.data, n,
                                           int(k), mn.ctypes.data, med.ctypes.data, avg.ctypes.data))
    return mn[:n], med[:n], avg[:n]


class RefSet:
    """Reference gene set on the device (t4_refset_create_from_fa: SeqSet::InputRefFa) and fastq-extractor's per-read
    predicate over it (t4_refset_scan: IsLowComplexity + SeqSet::HasHitInSet(read, 0))."""

    def __init__(self, fasta_path, k=9, lib: Lib | None = None, hit_len_required=27):
        self.lib = lib or default_lib()
        self.h = self.lib.refset_create_from_fa(fasta_path.encode(), int(k))
        if not self.h:
            raise T4Error(T4_E_INVAL, self.lib.err())
        self.k = k
        self.lib.check(self.lib.refset_set_hit_len_required(self.h, int(hit_len_required)))

    def close(self):
        if self.h:
            self.lib.refset_free(self.h)
            self.h = None

    def size(self):
        return self.lib.check(self.lib.refset_size(self.h))

    def names(self):
        return [self.lib.refset_name(self.h, i).decode() for i in range(self.size())]

    def seqset(self) -> "SeqSet":
        return _BorrowedSeqSet(self.k, self.lib, self.lib.refset_seqset(self.h))

    def set_radius(self, r):
        self.lib.check(self.lib.refset_set_radius(self.h, int(r)))

    def set_hit_len_required(self, v):
        self.lib.check(self.lib.refset_set_hit_len_required(self.h, int(v)))

    def get_overlaps(self, read, cap=4096):
        """SeqSet::GetOverlapsFromRead(read, 0, -1, 0, false) on the gene set: (n, int32[n, 8], similarity[n])."""
        out = np.zeros((cap, 8), dtype=np.int32)
        sim = np.zeros(cap, dtype=np.float64)
        n = self.lib.check(self.lib.refset_get_overlaps(self.h, read.encode(), out.ctypes.data, sim.ctypes.data, cap))
        if n < 0:
            return n, None, None
        return n, out[:n], sim[:n]

    def annotate(self, pool, seq_off, lens):
        """SeqSet::AnnotateRead(read, 0, ...) per read: (int32[n, 4, 8] for V, D, J, C; similarity float64[n, 4])."""
        pool = np.ascontiguousarray(pool)
        seq_off = np.ascontiguousarray(seq_off, dtype=np.uint64)
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        n = len(lens)
        out = np.zeros((max(1, n), 4, 8), dtype=np.int32)
        sim = np.zeros((max(1, n), 4), dtype=np.float64)
        self.lib.check(self.lib.refset_annotate(self.h, pool.ctypes.data, pool.nbytes, seq_off.ctypes.data, lens.ctypes.data, n,
                                                out.ctypes.data, sim.ctypes.data))
        return out[:n], sim[:n]

    def scan(self, pool, seq_off, lens):
        """(strand int8[n] = HasHitInSet(read, 0), low uint8[n] = IsLowComplexity(read), stats)."""
        pool = np.ascontiguousarray(pool)
        seq_off = np.ascontiguousarray(seq_off, dtype=np.uint64)
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        n = len(lens)
        strand = np.zeros(max(1, n), dtype=np.int8)
        low = np.zeros(max(1, n), dtype=np.uint8)
        st = np.zeros(2, dtype=np.uint64)
        self.lib.check(self.lib.refset_scan(self.h, pool.ctypes.data, pool.nbytes, seq_off.ctypes.data, lens.ctypes.data, n,
                                            strand.ctypes.data, low.ctypes.data, st.ctypes.data))
        return strand[:n], low[:n], dict(with_hit=int(st[0]), low_complexity=int(st[1]))


def sort_reads(pool, seq_off, lens, ids, min_cnt, median_cnt, avg_cnt, lib: Lib | None = None):
    """t4_sort_reads: the permutation std::sort(sortedReads) applies (main.cpp:1078).  ids: list of bytes / str."""
    lib = lib or default_lib()
    pool = np.ascontiguousarray(pool)
    seq_off = np.ascontiguousarray(seq_off, dtype=np.uint64)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    n = len(lens)
    idb = [i if isinstance(i, bytes) else i.encode() for i in ids]
    id_off = np.zeros(n + 1, dtype=np.uint64)
    id_off[1:] = np.cumsum([len(i) for i in idb])
    id_pool = np.frombuffer(b"".join(idb) + b"\0" * 16, dtype=np.uint8).copy()
    order = np.zeros(max(1, n), dtype=np.int64)
    lib.check(lib.sort_reads(pool.ctypes.data, pool.nbytes, seq_off.ctypes.data, lens.ctypes.data, id_pool.ctypes.data, id_pool.nbytes,
                             id_off.ctypes.data, np.ascontiguousarray(min_cnt, dtype=np.int32).ctypes.data,
                             np.ascontiguousarray(median_cnt, dtype=np.int32).ctypes.data,
                             np.ascontiguousarray(avg_cnt, dtype=np.float32).ctypes.data, n, order.ctypes.data))
    return order[:n]


def sort_reads_barcode(pool, seq_off, lens, ids, min_cnt, median_cnt, avg_cnt, barcode, barcode_min_cnt, lib: Lib | None = None):
    """t4_sort_reads_barcode: the permutation of std::sort(sortedReads, CompReadWithBarcode) (main.cpp:128-136) -- barcode
    ascending, barcodeMinCnt descending, then sort_reads' order.  Barcodes must be >= 0."""
    lib = lib or default_lib()
    pool = np.ascontiguousarray(pool)
    seq_off = np.ascontiguousarray(seq_off, dtype=np.uint64)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    n = len(lens)
    idb = [i if isinstance(i, bytes) else i.encode() for i in ids]
    id_off = np.zeros(n + 1, dtype=np.uint64)
    id_off[1:] = np.cumsum([len(i) for i in idb])
    id_pool = np.frombuffer(b"".join(idb) + b"\0" * 16, dtype=np.uint8).copy()
    order = np.zeros(max(1, n), dtype=np.int64)
    arrs = [np.ascontiguousarray(a, dtype=t) for a, t in ((min_cnt, np.int32), (median_cnt, np.int32), (avg_cnt, np.float32),
                                                          (barcode, np.int32), (barcode_min_cnt, np.int32))]
    lib.check(lib.sort_reads_barcode(pool.ctypes.data, pool.nbytes, seq_off.ctypes.data, lens.ctypes.data, id_pool.ctypes.data, id_pool.nbytes,
                                     id_off.ctypes.data, *[a.ctypes.data for a in arrs], n, order.ctypes.data))
    return order[:n]


ASSIGN_NOT_LISTED = -2


class Assign:
    """The AssignRead pass of the stage-1 driver over finished sets (t4_streams_assign_reads; main.cpp:2047-2118):
    extended sets built from the stage-1 sets, AssignRead of every assembled read of the workload, RecomputePosWeight."""

    def __init__(self, sets, wl: Workload, desc_off, kmer_length=17, n_workers=0, cuda_stream=None):
        self.lib = wl.lib
        self.n = int(desc_off[len(sets)])
        off = np.ascontiguousarray(desc_off, dtype=np.int64)
        hs = (C.c_void_p * len(sets))(*[s.h if isinstance(s, SeqSet) else s for s in sets])
        self.h = self.lib.streams_assign_reads(hs, len(sets), wl.h, off.ctypes.data, int(kmer_length), int(n_workers), cuda_stream)
        if not self.h:
            raise T4Error(T4_E_CUDA, self.lib.err())
        self.n_sets = len(sets)
        self.kmer_length = kmer_length

    def close(self):
        if self.h:
            self.lib.assign_free(self.h)
            self.h = None

    def results(self):
        """(assign int32[n, 8], similarity float64[n]) per record of the workload."""
        a = np.zeros((max(1, self.n), 8), dtype=np.int32)
        s = np.zeros(max(1, self.n), dtype=np.float64)
        self.lib.check(self.lib.assign_results(self.h, a.ctypes.data, s.ctypes.data))
        return a[:self.n], s[:self.n]

    def stats(self):
        s = np.zeros(4, dtype=np.uint64)
        self.lib.check(self.lib.assign_stats(self.h, s.ctypes.data))
        return dict(reads=int(s[0]), assign_calls=int(s[1]), assigned=int(s[2]), workers=int(s[3]))

    def extended_set(self, j) -> "SeqSet":
        h = self.lib.assign_extended_set(self.h, j)
        if not h:
            raise T4Error(T4_E_INVAL, self.lib.err())
        return _BorrowedSeqSet(self.kmer_length, self.lib, h)


class _BorrowedSeqSet(SeqSet):
    """A set owned by another object (t4_assign): same calls, never destroyed from here."""

    def close(self):
        self.h = None


SHARD_RANK, SHARD_BARCODE, SHARD_GENE = 0, 1, 2


def shard_reads(descs, n_streams, mode=SHARD_GENE, lib=None):
    """t4_shard_reads: (desc_off[S+1], records in stream order, order[new] = old index).  Host-only, no device needed."""
    lib = lib or default_lib()
    d = np.ascontiguousarray(descs).copy()
    n = len(d)
    off = np.zeros(max(1, min(n_streams, max(n, 1))) + 1, dtype=np.int64)
    order = np.zeros(max(n, 1), dtype=np.int64)
    S = lib.shard_reads(d.ctypes.data, n, int(n_streams), int(mode), off.ctypes.data, order.ctypes.data)
    if S < 0:
        lib.check(S)
    return off[:S + 1].copy(), d, order[:n]
