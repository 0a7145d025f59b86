/*
 * trust4_b200 -- C ABI of the H100-native (sm_90a) stage-1 assembly hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference has no FFI; its
 * boundary is the C++ class SeqSet as used by the stage-1 driver.  Every entry
 * point below names the reference interface it replaces (file:line under the
 * reference tree).  Plain pointers and sizes only; no torch / C++ types.
 *
 * One `t4_seqset` is one novel-contig set (reference: `SeqSet seqSet(k)`,
 * main.cpp:642) and, on the device, one *stream*: a persistent CTA owns its
 * contigs, posWeight columns and k-mer postings in HBM and executes the reads
 * submitted to it strictly in order (the reference's AddRead loop is serial,
 * main.cpp:1583-1880).  Many seqsets run concurrently, one CTA each.
 *
 * Return conventions follow the reference: AddRead >= 0 contig slot, -1 not
 * added, -2 overlapped but could not extend (SeqSet.hpp:3422-3425, 4463-4467).
 * Errors of this library are < T4_E_BASE and never abort the process.
 */
#ifndef TRUST4_B200_H
#define TRUST4_B200_H

#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#ifdef __cplusplus
extern "C" {
#endif

#define T4_OK 0
#define T4_E_BASE (-16)
#define T4_E_CUDA (-17)        /* CUDA runtime error (see t4_last_error) */
#define T4_E_NOMEM (-18)       /* device arena exhausted */
#define T4_E_INVAL (-19)       /* bad argument */
#define T4_E_UNSUPPORTED (-20) /* e.g. isLongSeqSet, read longer than T4_MAX_READ_LEN */
#define T4_E_NODEVICE (-21)    /* no CUDA device: there is NO CPU fallback */
#define T4_E_INTERNAL (-22)    /* device-side invariant violated */

#define T4_MAX_READ_LEN 512    /* device-side read length limit; longer reads return T4_E_UNSUPPORTED */

typedef struct t4_seqset t4_seqset;

/* ---- library / device ------------------------------------------------- */
/* Select the device and size the device arena (bytes; 0 = 1/2 of free HBM).
 * Optional: the first t4_seqset_create() calls t4_init(current device, 0). */
int t4_init(int device, size_t arena_bytes);
int t4_shutdown(void);
const char *t4_last_error(void);
const char *t4_version(void);
/* Bytes of device arena in use / capacity (diagnostics). */
int t4_arena_stats(size_t *used, size_t *capacity);
/* Drop every seqset at once (the arena is a bump allocator; all t4_seqset handles become stale). */
int t4_reset(void);

/* ---- SeqSet mirror ---------------------------------------------------- */
/* SeqSet::SeqSet(int kl), SeqSet.hpp:2558-2576 (radius 10, hitLenRequired 31,
 * novelSeqSimilarity 0.9, nomatchGapLimit from k). */
t4_seqset *t4_seqset_create(int kmer_length);
/* n sets with one device launch (read-sharded runs create thousands of streams). */
int t4_seqsets_create(int n, int kmer_length, t4_seqset **handles);
/* ... with SetHitLenRequired(l) and SetConsiderBarcodeInIndexHash(on) (SeqSet.hpp:2601, 2611; the driver sets them
 * once before the loop, main.cpp:1549-1565) applied to every new set by the same launch. */
int t4_seqsets_create_ex(int n, int kmer_length, int hit_len_required, int consider_barcode, t4_seqset **handles);
void t4_seqset_destroy(t4_seqset *s);
/* SeqSet::SetHitLenRequired, SeqSet.hpp:2601 */
int t4_seqset_set_hit_len_required(t4_seqset *s, int l);
/* SeqSet::SetNovelSeqSimilarity, SeqSet.hpp:2606 */
int t4_seqset_set_novel_seq_similarity(t4_seqset *s, double v);
/* SeqSet::SetConsiderBarcodeInIndexHash, SeqSet.hpp:2611.  As in the reference's KmerIndex (bucket
 * (code + barcode + 1) % 1000003, KmerIndex.hpp:29-33), two barcodes share one postings list per k-mer exactly when
 * barcode + 1 is equal modulo 1000003 (5 and 1000008; -1, i.e. no barcode, and 1000002): the >= 100-postings skip rule
 * of GetHitsFromRead sees the shared list's size, and a read without a barcode gets the hits on 1000002's contigs.
 * Needs k <= 15. */
int t4_seqset_set_consider_barcode_in_hash(t4_seqset *s, int on);
/* SeqSet::SetIsLongSeqSet, SeqSet.hpp:11082 -- only `0` is supported (reads <= 200 bp). */
int t4_seqset_set_is_long(t4_seqset *s, int on);
/* SeqSet::Size, SeqSet.hpp:2591 (counts released slots) */
int t4_seqset_size(t4_seqset *s);
int t4_seqset_kmer_length(t4_seqset *s);

/* int SeqSet::AddRead(char *read, char *geneName, int &strand, int barcode,
 *   int minKmerCount, bool repetitiveData, double similarityThreshold), SeqSet.hpp:3426 */
int t4_seqset_add_read(t4_seqset *s, const char *read, const char *gene_name, int *strand_inout,
                       int barcode, int min_kmer_count, int repetitive, double sim_threshold);
/* int SeqSet::RepeatAddRead(char *read), SeqSet.hpp:4477 */
int t4_seqset_repeat_add_read(t4_seqset *s, const char *read);
/* int SeqSet::InputNovelRead(const char *id, char *read, int strand, int barcode), SeqSet.hpp:3028 */
int t4_seqset_input_novel_read(t4_seqset *s, const char *id, const char *read, int strand, int barcode);
/* void SeqSet::UpdateAllConsensus(), SeqSet.hpp:4525 */
int t4_seqset_update_all_consensus(t4_seqset *s);
/* void SeqSet::ChangeKmerLength(int kl), SeqSet.hpp:4624 (compacts slots, rebuilds the index) */
int t4_seqset_change_kmer_length(t4_seqset *s, int kmer_length);
/* void SeqSet::ReleaseFinishedBarcodeSeq(std::map<int,int> barcodes, bool removeFromIndex, int contigMinCov,
 *   bool earlyStop), SeqSet.hpp:10815, as the stage-1 driver calls it (main.cpp:1855): one finished barcode,
 *   removeFromIndex = true, earlyStop = true. */
int t4_seqset_release_finished_barcode(t4_seqset *s, int barcode, int contig_min_cov);
/* void SeqSet::ReleaseShallowContigs(int minCov), SeqSet.hpp:10928 (main.cpp:1954) */
int t4_seqset_release_shallow_contigs(t4_seqset *s, int min_cov);
/* void SeqSet::InputNovelFa(char *filename), SeqSet.hpp:2986 (--debug-ns, main.cpp:711): every FASTA record becomes a
 * contig through InputNovelRead(id, seq, 1, -1).  Returns the number of records or a T4_E_* code. */
int t4_seqset_input_novel_fa(t4_seqset *s, const char *filename);
/* void SeqSet::Output(FILE*, std::vector<std::string>*), SeqSet.hpp:10939 */
int t4_seqset_output(t4_seqset *s, FILE *fp, const char *const *barcode_names, int n_barcode_names);
/* Same text into a malloc'ed buffer (caller frees with t4_free). */
int t4_seqset_output_mem(t4_seqset *s, char **buf, size_t *len);
void t4_free(void *p);

/* Contig accessors (hand contigs back to the CPU mate-extension code,
 * SeqSet::InputSeqSet consumer, SeqSet.hpp:3108).  Buffers may be NULL to query sizes.
 * Returns consensus length, or -1 for a released slot. */
int t4_seqset_get_contig(t4_seqset *s, int slot, char *consensus, int consensus_cap,
                         int32_t *pos_weight /* 4*len, [pos][ACGT] */, char *name, int name_cap,
                         int *barcode, int *num_read, int *min_left_ext_anchor, int *min_right_ext_anchor);

/* T4_CONTIG_PURGED: the contig was purged by ReleaseFinishedBarcodeSeq (reference: seqs[i].index == false and
 * posWeight compressed / freed; a host mirror re-applies that storage change, see integration/).  -1 for a released slot. */
#define T4_CONTIG_PURGED 1
int t4_seqset_contig_flags(t4_seqset *s, int slot);

/* int SeqSet::HasMotif(char *read, int strand), SeqSet.hpp:5029 (host utility) */
int t4_has_motif(const char *read, int strand);
/* void SeqSet::ReverseComplementInPlace(char*, int), SeqSet.hpp:2629 (host utility) */
void t4_reverse_complement_in_place(char *seq, int len);

/* ---- read-only probes over a frozen set (parity / roofline entry points) -- */
/* SeqSet::GetHitsFromRead + SortHits, SeqSet.hpp:1341, 1306.
 * Writes up to cap hits as int32[5] = {seqIdx, seqOffset, readOffset, strand, repeats},
 * ordered by (strand, seqIdx, readOffset, seqOffset).  Returns the hit count. */
int t4_seqset_get_hits(t4_seqset *s, const char *read, int strand, int barcode, int allow_total_skip,
                       int32_t *hits, int cap);
/* SeqSet::GetOverlapsFromRead (readType 0), SeqSet.hpp:1508: scored overlaps as
 * int32[8] = {seqIdx, readStart, readEnd, seqStart, seqEnd, strand, matchCnt, indelCnt}
 * plus similarity[i].  Returns the overlap count (or -1 when the read is shorter than k). */
int t4_seqset_get_overlaps(t4_seqset *s, const char *read, int strand, int barcode, int skip_repeats,
                           int32_t *overlaps, double *similarity, int cap);
/* AlignAlgo::GlobalAlignment_PosWeight, AlignAlgo.hpp:57: n independent problems on the device.
 * t_weights: concatenated int32[4] columns, p: concatenated chars; offsets arrays have n+1 entries.
 * align_out: concatenated edit strings, problem i at align_off[i] (capacity lent+lenp+1 each),
 * terminated by -1.  score_out[i] is the returned score. */
int t4_dp_pos_weight_batch(int n, const int32_t *t_weights, const int64_t *t_off, const char *p,
                           const int64_t *p_off, int8_t *align_out, const int64_t *align_off,
                           int32_t *score_out);

/* The same alignment through the two routines the stream kernel actually runs for its equal-length problems
 * (overhangs of ExtendOverlap, SeqSet.hpp:1165; same-diagonal gaps of GetOverlapsFromRead, SeqSet.hpp:1832-2006):
 * variant 0 = per-thread register banded DP, variant 1 = half-warp anti-diagonal DP (no <=2-mismatch fast path:
 * its caller settles those from popcounts), variant 2 = ExtendOverlap's overhang pass: problems 2k and 2k+1 run on the
 * two halves of one warp as a left overhang (statistics taken from its end) and a right one, and instead of the edit
 * string align_out receives at align_off[i] (a multiple of 4, 16 bytes) four int32: the matches, mismatches and indels
 * of the alignment and its good-prefix length (SeqSet.hpp:1176-1224); score_out is not written.  Variants 1 and 2 exist
 * only in the CUDA build.  Problem i spans columns/bases off[i]..off[i+1) of both inputs. */
int t4_dp_hot_path_batch(int n, int variant, const int32_t *t_weights, const int64_t *off, const char *p,
                         int8_t *align_out, const int64_t *align_off, int32_t *score_out);

/* ---- batch / multi-stream entry (the throughput path) ------------------ */
/* One element per iteration of the reference's AddRead loop (main.cpp:1583-1880):
 * everything the loop derives from the pre-processing (rough annotation, k-mer
 * counts, sort) is precomputed by the host into this record; everything that
 * depends on the evolving contig set is decided on the device. */
typedef struct t4_read_desc {
    uint64_t seq_off;        /* offset of the read (ASCII ACGTN) in the read pool */
    int32_t len;             /* read length */
    int32_t barcode;         /* sortedReads[i].barcode, -1 = none */
    int32_t min_cnt;         /* sortedReads[i].minCnt (rescue threshold, main.cpp:1914-1923) */
    int32_t min_kmer_count;  /* AddRead argument (main.cpp:1700-1701) */
    double sim_threshold;    /* main.cpp:1676-1694 */
    int32_t name_id;         /* InputNovelRead name on failure (index into names), -1 = none */
    int32_t mate_idx;        /* sortedReads[i].mateIdx as an index into this array, -1 = none */
    int32_t eq_lo, eq_hi;    /* [eq_lo,eq_hi): maximal run of records with this read string (main.cpp:1814-1835) */
    uint32_t flags;          /* T4_RD_* */
    int8_t strand_in;        /* strand passed to AddRead (0 = unknown) */
    int8_t novel_strand;     /* strand passed to InputNovelRead (main.cpp:1743) */
    char gene4[4];           /* 4-char gene prefix passed as geneName, zero padded */
    int8_t pad_[2];
} t4_read_desc;

#define T4_RD_DUP (1u << 0)           /* same read+barcode as the previous record (main.cpp:1596) */
#define T4_RD_FILTERED (1u << 1)      /* V/D/J/C order or C-gene filter hit (main.cpp:1609-1654) */
#define T4_RD_NOVEL_ON_FAIL (1u << 2) /* anchored: InputNovelRead(names[name_id]) if AddRead<0 (main.cpp:1706-1745) */
#define T4_RD_MOTIF (1u << 3)         /* HasMotif(read, +-1) != 0 (main.cpp:1752) */
#define T4_RD_GOOD_PLUS (1u << 4)     /* main.cpp:1782-1808 evaluates to good when strand==+1 */
#define T4_RD_GOOD_MINUS (1u << 5)    /* ... when strand==-1 */
#define T4_RD_MOTIF_FORCED (1u << 6)  /* replay mode: take the motif path with strand = novel_strand */

typedef struct t4_run_cfg {
    int32_t has_barcode;           /* main.cpp hasBarcode: no periodic UpdateAllConsensus / k change */
    int32_t repetitive;            /* trimLevel > 1 (AddRead repetitiveData) */
    int32_t change_k_threshold;    /* changeKmerLengthThreshold, main.cpp:641,1567 (0 = never) */
    int32_t update_consensus_every;/* main.cpp:1862 (10000; 0 = never) */
    int32_t do_rescue;             /* run the rescue pass main.cpp:1897-1940 */
    int32_t first_read_len;        /* firstReadLen (rescue is skipped when > 200) */
    int32_t final_update;          /* UpdateAllConsensus after each pass (main.cpp:1881,1939) */
    int32_t release_barcodes;      /* hasBarcode && !keepMissingBarcode: purge a barcode's contigs once all of its reads
                                      were assembled (main.cpp:1846-1859 -> ReleaseFinishedBarcodeSeq, SeqSet.hpp:10815);
                                      the per-barcode totals are counted over this seqset's records (main.cpp:1572-1581) */
    int32_t contig_min_cov;        /* --contigMinCov (main.cpp:741): argument of the purge above */
    int32_t reserved_;
} t4_run_cfg;

/* Observationally equal to running the reference loop (main.cpp:1583-1881, and
 * 1897-1940 when cfg->do_rescue) over descs[0..n) on this seqset.
 * ret_codes[i]: addRet of iteration i; strands[i]: sortedReads[i].strand afterwards;
 * rescue_ret (may be NULL): n entries, addRet of the rescue pass or INT32_MIN if not rescued. */
int t4_seqset_add_reads_batch(t4_seqset *s, const t4_run_cfg *cfg, const t4_read_desc *descs, int n,
                              const char *read_pool, size_t read_pool_bytes,
                              const char *const *names, int n_names,
                              int32_t *ret_codes, int8_t *strands, int32_t *rescue_ret);

/* The same over many independent seqsets at once: one CTA per stream, one launch.
 * Stream j consumes descs[desc_off[j] .. desc_off[j+1]) (mate_idx / eq_* are
 * relative to desc_off[j]).  Host buffers; H2D/D2H are part of the call. */
int t4_streams_run(t4_seqset *const *sets, int n_sets, const t4_run_cfg *cfg,
                   const t4_read_desc *descs, const int64_t *desc_off,
                   const char *read_pool, size_t read_pool_bytes,
                   const char *const *names, int n_names,
                   int32_t *ret_codes, int8_t *strands, int32_t *rescue_ret);

/* Host-side read sharding (SURVEY.md 8e; no device work): which of at most n_streams independent SeqSets assembles
 * which records of the driver's sorted read list (main.cpp:1583 walks sortedReads in this order).  `descs` is
 * reordered in place into stream order (a stream keeps the sorted order of its records), eq_lo / eq_hi / mate_idx are
 * rewritten relative to the record's stream (a mate in another stream becomes -1: no hint), desc_off[0..S] receives
 * the stream boundaries and order[j] the original index of new record j (to map t4_workload_results back).  A run of
 * identical read strings is never split.  Returns S (1 <= S <= n_streams; empty streams are dropped) or < 0.
 *   T4_SHARD_RANK    contiguous blocks of the sorted list with equal predicted cost (abundance ranks stay together)
 *   T4_SHARD_BARCODE the same, and a cut never falls inside a barcode (10x data: barcodes are independent assemblies,
 *                    main.cpp:1846-1859)
 *   T4_SHARD_GENE    runs grouped by the gene of their rough annotation (names[name_id] of the run's first record),
 *                    groups cut / packed into streams of equal predicted cost: a clonotype's reads meet in one SeqSet
 *                    whatever their abundance (the reference shards --repseq input by V gene too, main.cpp:1224-1235) */
#define T4_SHARD_RANK 0
#define T4_SHARD_BARCODE 1
#define T4_SHARD_GENE 2
int t4_shard_reads(t4_read_desc *descs, int64_t n_descs, int n_streams, int mode, int64_t *desc_off, int64_t *order);

/* Device-resident variant used by bench.py's `value` leg: the workload is
 * uploaded once (t4_workload_upload), then t4_streams_run_resident() only
 * launches kernels on `cuda_stream` (a cudaStream_t cast to void*, NULL = default). */
typedef struct t4_workload t4_workload;
t4_workload *t4_workload_upload(const t4_read_desc *descs, int64_t n_descs, const char *read_pool,
                                size_t read_pool_bytes, const char *const *names, int n_names);
void t4_workload_free(t4_workload *w);
int t4_streams_run_resident(t4_seqset *const *sets, int n_sets, const t4_run_cfg *cfg,
                            t4_workload *w, const int64_t *desc_off, void *cuda_stream);
/* Copy results of the last resident run back. */
int t4_workload_results(t4_workload *w, int32_t *ret_codes, int8_t *strands, int32_t *rescue_ret);
/* Which SeqSet calls each iteration of the loop made (what a call trace of the reference driver would show), one byte
 * per record: lets a host driver that keeps the reference's own loop replay the device's decisions call by call
 * (integration/t4_seqset_adapter.hpp, batch mode) and lets tests compare call sequences. */
#define T4_EV_ADD_READ (1u << 0)        /* AddRead was called (main.cpp:1700) */
#define T4_EV_REPEAT (1u << 1)          /* RepeatAddRead (main.cpp:1766) */
#define T4_EV_NOVEL_ANCHORED (1u << 2)  /* InputNovelRead with the gene name (main.cpp:1742) */
#define T4_EV_NOVEL_MOTIF (1u << 3)     /* InputNovelRead("Novel") after a good mate + motif (main.cpp:1752) */
#define T4_EV_CHANGE_K (1u << 4)        /* ChangeKmerLength after this iteration (main.cpp:1874-1879) */
#define T4_EV_RESCUED (1u << 5)         /* AddRead of the rescue pass (main.cpp:1926) */
#define T4_EV_PURGED (1u << 6)          /* ReleaseFinishedBarcodeSeq after this iteration (main.cpp:1855) */
int t4_workload_events(t4_workload *w, uint8_t *events);

/* Merge step (SURVEY.md 8e) and stage-1 product: pack every live contig of the given sets, in (set, slot) order, into ONE
 * caller-provided DEVICE buffer (e.g. a torch tensor) ready for an NCCL all-gather or one D2H copy.  Record = 32-byte
 * header {u32 set, slot, len, nameLen; i32 barcode, numRead; u32 recordBytes, flags} + consensus[len] + posWeight
 * columns [len][4] as u16 (flags bit 0, when every count of the contig fits 16 bits) or int32 + name, padded to 16 B.
 * With dev_buf == NULL only *bytes_needed / *n_contigs are computed. */
int t4_streams_pack_contigs(t4_seqset *const *sets, int n_sets, void *dev_buf, size_t cap, size_t *bytes_needed,
                            int64_t *n_contigs);

/* First device-side error among the streams (0 = none); details in t4_last_error(). */
int t4_streams_error(t4_seqset *const *sets, int n_sets);
/* Diagnostics: SM clock cycles the last op spent on each stream (load-balance analysis). */
int t4_streams_cycles(t4_seqset *const *sets, int n_sets, uint64_t *cycles);
/* Test hook: number of postings in the k-mer index and an order-independent checksum of them. */
int64_t t4_seqset_index_checksum(t4_seqset *s, uint64_t *checksum);
/* Test hook: checks the equality byte the engine keeps beside every posWeight column of every live contig against the
 * column; returns the number of columns checked, *bad the number whose byte is not IsBaseEqual of the column. */
int64_t t4_test_check_eq_bytes(t4_seqset *s, int64_t *bad);

/* Device counters accumulated since the last t4_reset()/probe (summed over streams):
 * [0] reads processed, [1] overhang DPs (ExtendOverlap), [2] k-mer lookups executed, [3] postings read (sum c_j),
 * [4] hits emitted (sum c_j'), [5] packed read bytes ceil(L/4), [6] overlaps scored, [7] gap DPs,
 * [8..15] clock cycles per phase: other, probe, hit sort, chains, scoring, ExtendOverlap, decide+commit,
 * InputNovelRead/RepeatAddRead/consensus; [16] overlaps extended; [17..19] cycles inside ExtendOverlap (bit masks with
 * the settling of every side that needs no DP, the list of deferred sides, their DPs), [20] reads taking the lazy ExtendOverlap path; [21] ExtendOverlaps the decision loop still runs
 * on demand on its single thread (s_make_exact: overlaps it consults without a result), [22] the clock cycles they take;
 * [23] reserved. */
#define T4_N_COUNTERS 24
int t4_last_counters(uint64_t *counters /* T4_N_COUNTERS */);

/* ---- batch k-mer probe over frozen sets (the north-star "k-mer probe kernel") ----------------------------
 * SeqSet::GetHitsFromRead (SeqSet.hpp:1341-1501) + KmerIndex::Search (KmerIndex.hpp:104) for every record of an uploaded
 * workload against the set of its stream (record i belongs to set j iff desc_off[j] <= i < desc_off[j+1]; desc_off[0]
 * must be 0), with the record's strand_in and barcode.  The sets are only read: reads are independent, so this runs
 * one warp per read over the whole GPU (2-bit packed reads, one-sector directory probes, TMA-staged postings) instead of
 * one CTA per set.  Results stay on the device in `out` (hit keys + per-record offset/count); the launch is
 * asynchronous on cuda_stream.  Consumers: read-only passes over finished contigs (AssignRead, SeqSet.hpp:4632, is the
 * next one) and the roofline measurement of SURVEY.md 8d. */
typedef struct t4_hits t4_hits;
t4_hits *t4_hits_create(int64_t max_records, size_t max_hits);
void t4_hits_free(t4_hits *h);
int t4_streams_get_hits(t4_seqset *const *sets, int n_sets, t4_workload *w, const int64_t *desc_off,
                        int allow_total_skip, void *cuda_stream, t4_hits *out);
/* Totals of the last probe (synchronises): stats[0] hits written (sum c_j'), [1] lookups executed, [2] postings read
 * (sum c_j), [3] packed read bytes, [4] algorithmic bytes of SURVEY.md 8d with the 8-byte hit key really written,
 * [5] the same with the survey's nominal 16-byte hit, [6] records longer than T4_MAX_READ_LEN (skipped), [7] records.
 * Returns T4_E_NOMEM (and the needed key count in t4_last_error) when `max_hits` was too small. */
int t4_hits_stats(t4_hits *h, uint64_t stats[8]);
/* Hits of one record as int32[4] = {seqIdx, seqOffset, readOffset, strand}, in read-position order (forward pass
 * first); returns their number (may exceed cap).  *flags bit 0: some k-mer has more than 10000 postings. */
int t4_hits_fetch(t4_hits *h, int64_t record, int32_t *hits, int cap, int *flags);
/* Device pointers of the result for device-side consumers: u64 keys[], u64 hit_off[records], u32 hit_cnt[records]. */
int t4_hits_device_buffers(t4_hits *h, void **keys, void **hit_off, void **hit_cnt);

/* ---- AssignRead pass over the finished sets (SURVEY.md 8f-2; the reference's second largest stage-1 cost) ----------
 * What the stage-1 driver does after the assembly for paired-end bulk data (main.cpp:2047-2118):
 *   SeqSet extendedSeq(k); extendedSeq.InputSeqSet(seqSet, false);      SeqSet.hpp:3108  (k = max(17, indexKmerLength))
 *   extendedSeq.SetNovelSeqSimilarity(0.95);
 *   for every assembled read, in the driver's order (main pass, then the rescued reads; main.cpp:1779, 1933):
 *       extendedSeq.AssignRead(read, strand, barcode, assign)           SeqSet.hpp:4632  (threads: AssignReads_Thread, main.cpp:607)
 *       -- a read whose string equals its predecessor's in that list keeps the predecessor's result (main.cpp:2078-2081)
 *   extendedSeq.SetNovelSeqSimilarity(0.9); extendedSeq.RecomputePosWeight(assembledReads)   SeqSet.hpp:4705
 * for every stage-1 set j = 0..n_sets-1 and the records desc_off[j]..desc_off[j+1] of the workload it assembled (the
 * results of the last t4_streams_run_resident on `w` say which reads were assembled and with which strand).
 * AssignRead only reads the set, so the reads are spread over `n_workers` CTAs of the whole GPU (0 = one resident wave),
 * whatever set they belong to.  Asynchronous on cuda_stream; the accessors below synchronise.  NULL on failure. */
typedef struct t4_assign t4_assign;
t4_assign *t4_streams_assign_reads(t4_seqset *const *sets, int n_sets, t4_workload *w, const int64_t *desc_off,
                                   int kmer_length, int n_workers, void *cuda_stream);
void t4_assign_free(t4_assign *a);
/* Per RECORD of the workload: assign[8*i] = {seqIdx, readStart, readEnd, seqStart, seqEnd, strand, matchCnt, 0} and
 * similarity[i] -- the fields of `struct _overlap` AssignRead returns (SeqSet.hpp:1248-1256).  seqIdx >= 0: slot in the
 * extended set; -1: AssignRead found no contig (the reference leaves the other fields stale then; here they are 0);
 * T4_ASSIGN_NOT_LISTED: the read was not assembled and is not part of the pass.  Either pointer may be NULL. */
#define T4_ASSIGN_NOT_LISTED (-2)
int t4_assign_results(t4_assign *a, int32_t *assign, double *similarity);
/* stats[0] reads in the pass, [1] AssignRead calls made (identical neighbours share one), [2] reads assigned to a
 * contig, [3] worker CTAs used. */
int t4_assign_stats(t4_assign *a, uint64_t stats[4]);
/* extendedSeq of set j after RecomputePosWeight (owned by `a`; valid until t4_reset / t4_assign_free): feed it to
 * t4_seqset_output / t4_seqset_get_contig, or on to the CPU mate-extension code (SeqSet::ExtendSeqFromReads). */
t4_seqset *t4_assign_extended_set(t4_assign *a, int j);
/* Device pointers of the two result arrays above, for device-side consumers. */
int t4_assign_device_buffers(t4_assign *a, void **assign, void **similarity);

/* ---- canonical k-mer counts and per-read count statistics (SURVEY.md 8f-3: the counting part of the pre-processing) --
 * KmerCount kmerCount(k); kmerCount.AddCount(read) for every read (KmerCount.hpp:64-97; main.cpp:404-440), then
 * kmerCount.GetCountStatsAndTrim(read, qual, minCnt, medianCnt, avgCnt) for every read (KmerCount.hpp:177-288;
 * main.cpp:981-1010): with qualities (--trimLevel >= 1, the default) the low-quality tail behind the last k-mer seen more
 * than once is cut first (new_len[i]: what is left, 0 = the driver drops the read), then min / median / average of the
 * counts of the read's canonical k-mers (a k-mer with an N does not count; no valid k-mer: -len; shorter than k: -1; any
 * N: min 0).  These numbers order the reads (main.cpp:103-125) and pick the AddRead thresholds (main.cpp:1675-1694).
 * Host buffers; record i is read_pool[seq_off[i] .. seq_off[i] + len[i]) and qual_pool at the same offsets (NULL = the
 * qual == NULL call of --trimLevel 0).  Any output may be NULL. */
int t4_kmer_count_stats(const char *read_pool, const char *qual_pool, size_t pool_bytes, const uint64_t *seq_off,
                        const int32_t *len, int64_t n, int kmer_length, int32_t *min_cnt, int32_t *median_cnt,
                        float *avg_cnt, int32_t *new_len);
/* The same on DEVICE buffers (all pointers; qual / new_len may be NULL; `table` = scratch of
 * t4_kmer_count_table_bytes(capacity hint, at most the total number of k-mer instances) bytes), asynchronous on
 * cuda_stream: two launches of t4_kcount_kernel (count, statistics). */
size_t t4_kmer_count_table_bytes(int64_t n_kmer_instances);
int t4_kmer_count_stats_device(const void *read_pool, const void *qual_pool, const void *seq_off, const void *len, int64_t n,
                               int kmer_length, void *table, size_t table_bytes, void *min_cnt, void *median_cnt,
                               void *avg_cnt, void *new_len, void *cuda_stream);
/* stats[0] k-mers counted, [1] distinct k-mers, [2] table slots, [3] 1 = table overflow (results invalid), 2 = a barcode
 * outside [0, barcode_max] (t4_barcode_kmer_count_stats_device; results invalid).  Synchronises. */
int t4_kmer_count_table_stats(const void *table, size_t table_bytes, uint64_t stats[4]);
/* The barcode-wise statistics of a --barcode run (main.cpp:1128-1180; threaded: BarcodeKmerCount_Thread, main.cpp:569-604):
 * for every barcode a fresh KmerCount(21, 23) gets AddCount(read) of the reads of that barcode, then
 * GetCountStatsAndTrim(read, NULL, barcodeMinCnt, barcodeMedianCnt, barcodeAvgCnt) for each of them (no quality trimming).
 * bc_*[i] are read i's numbers, exactly as above but over its own barcode's reads only.  Reads may come in any order:
 * one table keyed by (barcode, k-mer), one pass per 2^21 barcode ids that hold reads.  barcode[i] in [0, 2^31) (negative:
 * T4_E_INVAL); kmer_length <= 21 (else T4_E_INVAL); reads longer than T4_MAX_READ_LEN: T4_E_UNSUPPORTED; a table
 * overflow: T4_E_INTERNAL.  Host buffers; any output may be NULL.  Verified on an H100 against the reference. */
int t4_barcode_kmer_count_stats(const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len,
                                const int32_t *barcode, int64_t n, int kmer_length, int32_t *bc_min_cnt,
                                int32_t *bc_median_cnt, float *bc_avg_cnt);
/* The same on DEVICE buffers, asynchronous on cuda_stream: every barcode[i] must lie in [0, barcode_max] (one pass per
 * 2^21 ids up to barcode_max, two launches of t4_kcount_bc_kernel each); `table` as for t4_kmer_count_stats_device.
 * t4_kmer_count_table_stats afterwards tells whether the results are valid. */
int t4_barcode_kmer_count_stats_device(const void *read_pool, const void *seq_off, const void *len, const void *barcode,
                                       int64_t n, int32_t barcode_max, int kmer_length, void *table, size_t table_bytes,
                                       void *bc_min_cnt, void *bc_median_cnt, void *bc_avg_cnt, void *cuda_stream);

/* ---- stage-0 candidate extraction against a reference gene set (SURVEY.md 8f-4: fastq-extractor's predicate) --------
 * `SeqSet refSet(k); refSet.InputRefFa(fasta)` (FastqExtractor.cpp:313-318; SeqSet.hpp:2673-2864 with isIMGT == false:
 * ids with "/OR" skipped except D genes, '.' removed, every character that is not an upper-case A/C/G/T becomes N,
 * identical sequences kept once with their names joined by '|') as one indexed set on the device.  Plain-text FASTA. */
typedef struct t4_refset t4_refset;
t4_refset *t4_refset_create_from_fa(const char *fasta_path, int kmer_length);
void t4_refset_free(t4_refset *r);
int t4_refset_size(t4_refset *r);                      /* sequences kept */
const char *t4_refset_name(t4_refset *r, int i);       /* SeqSet::GetSeqName */
t4_seqset *t4_refset_seqset(t4_refset *r);             /* the set itself (owned by r), e.g. for t4_seqset_get_hits */
int t4_refset_set_hit_len_required(t4_refset *r, int l); /* SeqSet::SetHitLenRequired, FastqExtractor.cpp:455 (27, or 23, or readLen / 5) */
int t4_refset_set_radius(t4_refset *r, int radius);      /* SeqSet::SetRadius, SeqSet.hpp:2596 (default 10) */
/* For every read: low_complexity_out[i] = IsLowComplexity(read) (FastqExtractor.cpp:106-127) and strand_out[i] =
 * refSet->HasHitInSet(read, 0) (SeqSet.hpp:3144-3327: 0 no hit, +1 / -1 the strand of the best chain of seed hits on one
 * gene -- buckets per (strand, gene), GetOverlapsFromHits with the reference-sequence rules: diagonal windows of `radius`,
 * longest increasing subsequence, hit length on read and gene >= hitLenRequired).  fastq-extractor keeps a read (pair)
 * iff `!low && strand != 0` for the read or its mate (IsGoodCandidate, FastqExtractor.cpp:129-134, 211-219).
 * Host buffers; stats (may be NULL): [0] reads with a hit, [1] low-complexity reads. */
int t4_refset_scan(t4_refset *r, const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len,
                   int64_t n, int8_t *strand_out, uint8_t *low_complexity_out, uint64_t stats[2]);
/* SeqSet::GetOverlapsFromRead(read, 0, -1, 0, false, overlaps) on the gene set -- the call SeqSet::AnnotateRead makes per
 * read (SeqSet.hpp:6050), first half of the rough annotation (SURVEY.md 8f-1): chains with the reference-sequence rules
 * (or the V-end / J-start rescue, GetVJOverlapsFromHits), gaps scored by the affine AlignAlgo::GlobalAlignment, indels
 * allowed, similarity >= 0.75.  Same output layout as t4_seqset_get_overlaps.  Verified on an H100 against the reference.
 * A read with more seed hits than the per-read work space (65 536) returns T4_E_NOMEM; later calls are not affected. */
int t4_refset_get_overlaps(t4_refset *r, const char *read, int32_t *overlaps, double *similarity, int cap);
/* SeqSet::AnnotateRead(read, 0, geneOverlap, NULL, NULL) for n reads -- the rough annotation of the stage-1 driver
 * (main.cpp:1084-1120; SeqSet.hpp:6016-6340, detailLevel 0): contig intervals of the read (runs of N's), the overlaps of
 * every interval (above), the best gene per type with similarity >= 0.8, one cell type and chain per read, the check for a
 * random short constant-gene match.  gene_overlaps[i][t][8] for t = V, D, J, C = {seqIdx (-1: none), readStart, readEnd,
 * seqStart, seqEnd, strand, matchCnt, indelCnt}; similarity[i][t].  Host buffers.  Verified on an H100 against the
 * reference.  A batch with a read over the per-read hit limit returns T4_E_NOMEM as a whole; later calls are not affected. */
int t4_refset_annotate(t4_refset *r, const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len,
                       int64_t n, int32_t *gene_overlaps, double *similarity);
/* std::sort(sortedReads.begin(), sortedReads.end()) of the stage-1 driver (main.cpp:1078) with _sortRead::operator<
 * (main.cpp:103-125: minCnt, medianCnt, avgCnt, length descending, then read string and id ascending): order[j] = index of
 * the j-th record.  Host buffers; ids are id_pool[id_off[i] .. id_off[i+1]).  A merge sort of independent binary searches
 * on the device.  Verified on an H100 against the reference. */
int t4_sort_reads(const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len, const char *id_pool,
                  size_t id_pool_bytes, const uint64_t *id_off, const int32_t *min_cnt, const int32_t *median_cnt,
                  const float *avg_cnt, int64_t n, int64_t *order);
/* The read order of a --barcode run: std::sort with CompReadWithBarcode (main.cpp:128-136: barcode ascending,
 * barcodeMinCnt descending, then _sortRead::operator<).  The driver sorts by barcode while every barcodeMinCnt is still 0
 * (main.cpp:1126), counts per barcode, then re-sorts each barcode group (main.cpp:1183-1192); one call after
 * t4_barcode_kmer_count_stats gives the same sequence.  t4_sort_reads' arguments plus barcode[i] (>= 0: the comparator is
 * an order only then; a negative one gives T4_E_INVAL) and barcode_min_cnt[i].  Verified on an H100 against the reference. */
int t4_sort_reads_barcode(const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len,
                          const char *id_pool, size_t id_pool_bytes, const uint64_t *id_off, const int32_t *min_cnt,
                          const int32_t *median_cnt, const float *avg_cnt, const int32_t *barcode,
                          const int32_t *barcode_min_cnt, int64_t n, int64_t *order);
/* AlignAlgo::IsMateOverlap(fr, flen, sr, slen, minOverlap, offset, bestMatchCnt, checkTandem) (AlignAlgo.hpp:1027-1096)
 * for n read pairs, as ProcessRead calls it to detect read-through and overlapping mates (main.cpp:264, 291): overlap_size[i]
 * is the return value (-1: no unambiguous overlap), offset[i] / best_match_cnt[i] the two outputs as the function leaves them
 * (-1 when it never assigned them).  Host buffers.  Verified on an H100 against the reference. */
int t4_mate_overlap_batch(const char *read_pool, size_t pool_bytes, const uint64_t *f_off, const int32_t *f_len,
                          const uint64_t *s_off, const int32_t *s_len, const int32_t *min_overlap,
                          const uint8_t *check_tandem, int64_t n, int32_t *overlap_size, int32_t *offset,
                          int32_t *best_match_cnt);
/* Test hook, host only: SeqSet::LongestIncreasingSubsequence (SeqSet.hpp:342-474) exactly as the scan applies it to the
 * hits (a[i], b[i]) of a diagonal window sorted by b; returns the chain length, the chain in out_a / out_b (room for n). */
int t4_test_lis(const int32_t *a, const int32_t *b, int n, int32_t *out_a, int32_t *out_b);
/* The same on DEVICE buffers (ctrl: 64 bytes of device scratch; afterwards u64 ctrl[1] = reads with a hit, ctrl[2] =
 * low-complexity reads); n_workers CTAs (0 = one resident wave); asynchronous on cuda_stream. */
int t4_refset_scan_device(t4_refset *r, const void *read_pool, const void *seq_off, const void *len, int64_t n,
                          void *strand_out, void *low_complexity_out, void *ctrl, int n_workers, void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif
