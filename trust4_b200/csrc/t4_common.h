// Shared definitions of the stream engine: device-resident data layout and the
// build-mode macros.  The engine source (t4_engine.h) is written once against a
// (tid, nt, barrier) abstraction:
//   * product build (nvcc, sm_90a): one CTA per stream, T4_SYNC = __syncthreads();
//   * test-only emulation build (g++, -DT4_EMU): nt = 1, barriers are no-ops.  It
//     exists so the bit-exact logic can be debugged in a container without a GPU
//     (tests/emu); it is never linked into libtrust4_b200.so.
#ifndef T4_COMMON_H
#define T4_COMMON_H

#include <stdint.h>
#include <string.h>
#include "../../include/trust4_b200.h"

typedef uint64_t u64;
typedef uint32_t u32;
typedef int64_t i64;

#if defined(__CUDACC__) && !defined(T4_EMU)
#define T4_CUDA 1
#define T4_HD __host__ __device__
#define T4_D __device__
#define T4_SYNC() __syncthreads()
#define T4_SYNC_OR( x ) __syncthreads_or( x )
// Large collective routines with several call sites are real functions in the product build: inlined everywhere the
// stream kernel was 70 k SASS instructions (1.1 MB) and 18 % of its stall cycles were instruction fetch.
#ifdef T4_INLINE_ALL
#define T4_BIG inline
#else
#define T4_BIG __noinline__
#endif
#else
#define T4_BIG inline
#define T4_CUDA 0
#define T4_HD
#define T4_D
#define T4_SYNC() ((void)0)
#define T4_SYNC_OR( x ) ( x )
#endif

#define T4_DEV_MAX_READ T4_MAX_READ_LEN       /* device-side read length limit (reads > 200 bp make the reference switch to isLongSeqSet) */
#define T4_ALIGN 32               /* arena allocations are sector aligned: a postings list of <= 4 entries is ONE 32-byte sector */
#define T4_BIG_REPEAT 10000       /* SeqSet.hpp:799, 875, 937: hits[k].repeats <= 10000 */
#define T4_KINDEX_HASH_MAX 1000003u /* KmerIndex.hpp:21: buckets of the k-mer index; barcodes equal modulo it share postings lists */

// ---- key layout of a seed hit (one u64 per hit; SeqSet.hpp:53 `_hit` carries the same information) ----
// [63] strand (+1 -> 1, -1 -> 0) | [62:41] contig slot | [40:20] diagonal c = a - b + 2^20 | [19:1] contig offset b | [0] repeats > 10000
#define T4_KEY_STRAND_SHIFT 63
#define T4_KEY_IDX_SHIFT 41
#define T4_KEY_C_SHIFT 20
#define T4_KEY_B_SHIFT 1
#define T4_KEY_IDX_BITS 22
#define T4_KEY_C_BIAS (1 << 20)
#define T4_KEY_B_MASK ((1u << 19) - 1)
#define T4_KEY_C_MASK ((1u << 21) - 1)
#define T4_KEY_INVALID (~0ull)

struct T4Global            // arena header at offset 0
{
	u64 top ;              // bump pointer (bytes), device-side atomicAdd
	u64 cap ;
	u64 counters[T4_N_COUNTERS] ;
	u64 firstError ;       // first T4_E_* raised by any stream since the last reset: (u32)code | aux << 32; 0 = none
	u64 pad[5] ;
} ;

struct T4Dir               // one k-mer directory slot (32 B = one HBM sector); KmerIndex.hpp:20-116
{
	u64 key ;              // k-mer code (+ barcode salt) + 1; 0 = empty
	u64 listOff ;          // arena offset of the postings array (u64 each: idx<<32 | offset)
	u32 cnt ;
	u32 cap ;
	u32 lock ;
	u32 pad ;
} ;

struct T4Contig            // SeqSet.hpp:19 `_seqWrapper`, novel contigs only (isRef is always false in the stage-1 seqSet)
{
	u64 consOff ;          // char[cap], the consensus occupies [lead, lead + len)
	u64 pwOff ;            // int32[4][cap] per base, same lead, then u8[cap] equality bytes (t4_eq), same lead
	u64 nameOff ;
	int nameLen ;
	int len ;              // consensusLen; alive iff consOff != 0
	int cap ;
	int lead ;             // slack on the left: left extension is a pointer move, not a memmove
	int minLeftExtAnchor, minRightExtAnchor ;
	int barcode ;
	int numRead ;
	int flags ;            // T4_CF_*
	int packNarrow ;       // scratch of t4_streams_pack_contigs: 1 = every posWeight count of this contig fits 16 bits
} ;
#define T4_CF_NOINDEX 1    /* seqs[i].index == false: purged by ReleaseFinishedBarcodeSeq (SeqSet.hpp:10849) */

// bytes of one packed contig record (t4_streams_pack_contigs): 32-byte header + consensus + posWeight columns as 4 x u16
// (when all counts of the contig fit; the usual case, halves the merge exchange and the contig D2H) or 4 x i32 + name,
// padded to 16 bytes
T4_HD inline u64 t4_pack_record_bytes( const T4Contig &k )
{
	return ( 32ull + ( k.packNarrow ? 9ull : 17ull ) * k.len + k.nameLen + 15 ) & ~15ull ;
}

struct T4Ovl               // SeqSet.hpp:76 `_overlap`
{
	int seqIdx ;
	int readStart, readEnd ;
	int seqStart, seqEnd ;
	int strand ;
	int matchCnt ;
	int indelCnt ;
	double similarity ;
	int hcStart, hcCnt ;   // hitCoords = keys[hcStart .. hcStart+hcCnt) of the sorted hit array
	int preMatchCnt ;      // matchCnt before scoring (2*hitLen), consulted by the pre-filters SeqSet.hpp:1705-1794
	int infoFromHits ;
} ;

struct T4Stream            // one SeqSet (SeqSet.hpp:189-230 private members) + its scratch + loop state
{
	int kmerLength ;
	int radius ;
	int hitLenRequired ;
	int nomatchGapLimit ;
	int isLongSeqSet ;
	int considerBarcode ;
	double novelSeqSimilarity ;
	double repeatSimilarity ;
	// contigs
	int nSeqs, seqCap ;
	u64 seqsOff ;
	// k-mer directory
	u64 dirOff ;
	u32 dirCap, dirUsed ;
	// prevAddInfo (SeqSet.hpp:205)
	int prevSeqIdx, prevReadStart, prevReadEnd, prevSeqStart, prevStrand ;
	// scratch
	u64 keysAOff, keysBOff ;       // u64[hitCap] each
	u64 grpOff, runOff ;           // u32[hitCap + 1]
	u32 hitCap ;
	u64 keysROff, keysR2Off ;      // u64[hitCapR]: the hits once more in SortHits order, only when a k-mer has > 10000 postings
	u32 hitCapR ;
	u64 posOff ;                   // per read position scratch, see T4Pos
	u64 ovlOff, ovlTmpOff, extOff, failOff, anchorOff ;
	u64 bitsOff ;                  // u32[ovlCap * 32]: IsBaseEqual bit masks of the overhangs (ExtendOverlap)
	u32 ovlCap ;
	u64 dpOff ;                    // per-thread DP scratch, dpStride bytes each
	u32 dpStride ;
	int nThreads ;
	// driver-loop state (main.cpp:1530-1531, 640-641)
	int assembledReadCnt ;
	int prevAddRet ;
	int changeKThreshold ;
	int error ;                    // first T4_E_* raised on the device
	int errorAux ;
	// stream-local slab carved out of the arena (keeps small allocations off the global bump pointer)
	u64 slabTop, slabEnd ;
	// stats
	u64 nReads, nAddRead ;
} ;

struct T4Pos               // per (strand pass, read position) lookup record
{
	u64 listOff ;
	u64 code ;                     // rolling k-mer code ending at this position (N encoded as A)
	u32 cnt ;                      // postings of the k-mer (0 when the k-mer contains an N)
	u32 base ;                     // first hit slot, 0xffffffff = lookup not taken
} ;

// ---- contigs out of the arena: block bodies of t4_gather_kernel, t4_pack_size_kernel and t4_pack_kernel ----
// Contig c's payload into one contiguous buffer: [consensus len][posWeight 16*len][name nameLen] at out + outOff[c].
T4_D inline void t4_gather_block( char *A, const T4Contig *ct, const u64 *outOff, char *out, int n, int c, u32 tid, u32 nt )
{
	if ( c >= n || ct[c].consOff == 0 )
		return ;
	const T4Contig &k = ct[c] ;
	char *o = out + outOff[c] ;
	const char *cons = A + k.consOff + k.lead ;
	const char *pw = A + k.pwOff + 16ull * k.lead ;
	const char *nm = A + k.nameOff ;
	for ( int i = tid ; i < k.len ; i += nt )
		o[i] = cons[i] ;
	for ( int i = tid ; i < 16 * k.len ; i += nt )
		o[k.len + i] = pw[i] ;
	for ( int i = tid ; i < k.nameLen ; i += nt )
		o[17 * k.len + i] = nm[i] ;
}

// Stream j: decide for every live contig whether its posWeight counts fit 16 bits (scratch flag in the contig record),
// and sum the record sizes.
T4_D inline void t4_pack_size_block( char *A, const u64 *streamOff, u64 *sizes, u64 *counts, u32 j, u32 tid, u32 nt )
{
	const T4Stream *st = (const T4Stream *)( A + streamOff[j] ) ;
	T4Contig *ct = (T4Contig *)( A + st->seqsOff ) ;
	u64 tot = 0, n = 0 ;
	for ( int i = 0 ; i < st->nSeqs ; ++i )
	{
		T4Contig &k = ct[i] ;
		if ( !k.consOff )
			continue ;
		const int *pw = (const int *)( A + k.pwOff + 16ull * k.lead ) ;
		int wide = 0 ;
		for ( int x = tid ; x < 4 * k.len ; x += nt )
			wide |= ( (unsigned)pw[x] > 65535u ) ;
		wide = T4_SYNC_OR( wide ) ;
		if ( tid == 0 )
			k.packNarrow = wide ? 0 : 1 ;
		T4_SYNC() ;
		tot += t4_pack_record_bytes( k ) ;
		++n ;
	}
	if ( tid == 0 )
	{
		sizes[j] = tot ;
		counts[j] = n ;
	}
}

// Stream j's live contigs as packed records (t4_pack_record_bytes) from out + outOff[j] on.
T4_D inline void t4_pack_block( char *A, const u64 *streamOff, const u64 *outOff, char *out, u32 j, u32 tid, u32 nt )
{
	const T4Stream *st = (const T4Stream *)( A + streamOff[j] ) ;
	const T4Contig *ct = (const T4Contig *)( A + st->seqsOff ) ;
	u64 o = outOff[j] ;
	for ( int i = 0 ; i < st->nSeqs ; ++i )
	{
		const T4Contig &k = ct[i] ;
		if ( !k.consOff )
			continue ;
		u64 rb = t4_pack_record_bytes( k ) ;
		char *rec = out + o ;
		if ( tid == 0 )
		{
			u32 *h = (u32 *)rec ;
			h[0] = j ; h[1] = (u32)i ; h[2] = (u32)k.len ; h[3] = (u32)k.nameLen ;
			h[4] = (u32)k.barcode ; h[5] = (u32)k.numRead ; h[6] = (u32)rb ; h[7] = k.packNarrow ? 1u : 0u ;
		}
		const char *cons = A + k.consOff + k.lead ;
		const int *pw = (const int *)( A + k.pwOff + 16ull * k.lead ) ;
		const char *nm = A + k.nameOff ;
		for ( int x = tid ; x < k.len ; x += nt )
			rec[32 + x] = cons[x] ;
		u64 nameAt ;
		if ( k.packNarrow )
		{
			// the columns start at byte 32 + len (any alignment): byte stores
			unsigned char *d = (unsigned char *)rec + 32 + k.len ;
			for ( int x = tid ; x < 4 * k.len ; x += nt )
			{
				const unsigned v = (unsigned)pw[x] ;
				d[2 * x] = (unsigned char)( v & 255u ) ;
				d[2 * x + 1] = (unsigned char)( v >> 8 ) ;
			}
			nameAt = 32ull + 9ull * k.len ;
		}
		else
		{
			const char *pb = (const char *)pw ;
			for ( int x = tid ; x < 16 * k.len ; x += nt )
				rec[32 + k.len + x] = pb[x] ;
			nameAt = 32ull + 17ull * k.len ;
		}
		for ( int x = tid ; x < k.nameLen ; x += nt )
			rec[nameAt + x] = nm[x] ;
		// tail padding of the 16-byte aligned record: defined bytes (the all-gathered buffers are compared bytewise)
		for ( u64 x = nameAt + k.nameLen + tid ; x < rb ; x += nt )
			rec[x] = 0 ;
		o += rb ;
	}
}

// ---- 2-bit packed reads (KmerCode.hpp:94-109 semantics on words) ----
// A read of `len` bases occupies t4_pack_words(len) u64 words, W = ceil(len / 32):
//   fw[W]  forward strand, base j in bits [63 - 2 (j & 31) - 1, 63 - 2 (j & 31)] of word j >> 5 (first base most
//          significant, like KmerCode::Append shifting left), A 0 C 1 G 2 T 3, N stored as 00;
//   rc[W]  the reverse complement in the same layout (N stays N: 00);
//   nm[ceil(W/2)] u64 = u32[W]: bit (j & 31) of word j >> 5 set iff forward base j is 'N'.
// A k-mer is then one funnel shift of two words; its validity window (KmerCode::IsValid) is k bits of the N mask.
T4_HD inline u32 t4_pack_w( int len ) { return (u32)( len + 31 ) >> 5 ; }
T4_HD inline u32 t4_pack_words( int len ) { u32 W = t4_pack_w( len ) ; return 2 * W + ( ( W + 1 ) >> 1 ) ; }

// Word w of a packed read: 32 forward bases, 32 reverse-complement bases, 32 mask bits.  *odd is set when a base is
// none of ACGTN (the packed form cannot carry it: such workloads keep assembling from the ASCII pool).
T4_HD inline int t4_nuc2( char c ) { return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : c == 'N' ? 0 : 3 ; }
T4_HD inline void t4_pack_word( const char *s, int len, int w, u64 *fw, u64 *rc, u32 *nm, u32 *odd )
{
	u64 f = 0, b = 0 ;
	u32 mk = 0 ;
	for ( int i = 0 ; i < 32 ; ++i )
	{
		const int j = 32 * w + i ;
		if ( j >= len )
			break ;
		const char c = s[j] ;
		if ( c == 'N' )
			mk |= 1u << i ;
		else
		{
			if ( c != 'A' && c != 'C' && c != 'G' && c != 'T' )
				*odd = 1 ;
			f |= (u64)t4_nuc2( c ) << ( 62 - 2 * i ) ;
		}
		const char cr = s[len - 1 - j] ; // reverse-complement base j (SeqSet::ReverseComplement, SeqSet.hpp:2616)
		if ( cr != 'N' )
			b |= (u64)( 3 - t4_nuc2( cr ) ) << ( 62 - 2 * i ) ;
	}
	*fw = f ;
	*rc = b ;
	*nm = mk ;
}

// ASCII pool -> 2-bit packed pool (t4_pack_reads_kernel): item g = word g % wMax of read g / wMax.  *odd is set when a
// read holds a character outside ACGTN (the packed form cannot represent it; callers then keep using the ASCII pool).
struct T4PackReadsParams
{
	const t4_read_desc *descs ;
	i64 n ;
	const char *pool ;
	u64 packStride ;               // u64 words per record
	int wMax ;                     // words of the longest read
	u64 *packed ;
	u32 *odd ;
} ;

T4_HD inline void t4_pack_read_word( const T4PackReadsParams &P, i64 g )
{
	const i64 r = g / P.wMax ;
	const int w = (int)( g % P.wMax ) ;
	if ( r >= P.n )
		return ;
	const int len = P.descs[r].len ;
	if ( len <= 0 || len > T4_DEV_MAX_READ )
		return ;
	const int W = (int)t4_pack_w( len ) ;
	if ( w >= W )
		return ;
	u64 *fw = P.packed + (u64)r * P.packStride, *rc = fw + W ;
	u32 *nm = (u32 *)( fw + 2 * W ) ;
	t4_pack_word( P.pool + P.descs[r].seq_off, len, w, fw + w, rc + w, nm + w, P.odd ) ;
	if ( w == 0 && ( W & 1 ) )
		nm[W] = 0 ;
}

// Pointers to buffers outside the arena (workloads, staging, outputs) are absolute addresses stored in u64.
template <class T> T4_HD inline T *t4_x( u64 p ) { return (T *)(uintptr_t)p ; }

struct T4Names             // gene-name table of a workload (absolute pointers)
{
	u64 pool ;                     // char[]
	u64 off ;                      // u32[n+1]
	int n ;
	int pad ;
} ;

// One op of the stream kernel.
enum
{
	T4_OP_NONE = 0,
	T4_OP_ADD_READ,
	T4_OP_REPEAT,
	T4_OP_INPUT_NOVEL,
	T4_OP_UPDATE_ALL,
	T4_OP_CHANGE_K,
	T4_OP_GET_HITS,
	T4_OP_GET_OVERLAPS,
	T4_OP_RUN_LOOP,
	T4_OP_UNUSED_,
	T4_OP_INIT,
	T4_OP_RELEASE_BARCODE,
	T4_OP_RELEASE_SHALLOW,
	// auxiliary kernel (t4_assign.h): the AssignRead pass over frozen sets
	T4_OP_ASSIGN_PREP,
	T4_OP_ASSIGN,
	T4_OP_ASSIGN_RECOMPUTE,
	// ... and the stage-0 scan against a reference gene set (t4_refscan.h)
	T4_OP_REF_INPUT,
	T4_OP_REF_SCAN,
	// t4_annot_kernel (t4_annot.h): GetOverlapsFromRead on a reference gene set
	T4_OP_REF_OVERLAPS,
	T4_OP_REF_ANNOTATE,
} ;

struct T4Op                // per-CTA launch record
{
	u64 streamOff ;                // arena offset of the T4Stream
	int op ;
	int n ;                        // RUN_LOOP: number of descs
	u64 desc ;                     // t4_read_desc[n]            (absolute)
	u64 pool ;                     // read pool                  (absolute)
	u64 names ;                    // T4Names                    (absolute)
	u64 retCodes, strands, rescueRet ; // outputs int32[n], int8[n], int32[n] (absolute)
	u64 rescueList ;               // int32[n] scratch
	u64 good ;                     // int8[n] goodCandidate
	u64 info ;                     // int32[n]
	u64 events ;                   // uint8[n] T4_EV_* of every loop iteration (absolute), 0 = not recorded
	u64 packed ;                   // 2-bit packed reads of this op's records (absolute; record i at packed + i * packStride words), 0 = ASCII pool
	u64 packStride ;               // u64 words per record
	t4_run_cfg cfg ;
	// single-call ops
	u64 read ;                     // char[len] (absolute)
	int len ;
	int strand ;
	int barcode ;
	int minKmerCount ;
	int repetitive ;
	int kl ;
	double thr ;
	char gene[8] ;
	u64 name ; int nameLen ; int pad0 ;
	u64 out ;                      // GET_HITS / GET_OVERLAPS output buffer (absolute)
	int outCap ;
	int ret ;                      // result
	int strandOut ;
	int pad1 ;
	u64 out2 ;
	u64 stat0, stat1 ;
} ;

struct T4InitParams        // T4_OP_INIT: lay out and initialise a fresh stream at streamOff
{
	int kmerLength ;
	int nomatchGapLimit ;
	int nThreads ;
	u32 seqCap, dirCap, hitCap, ovlCap ;
	u32 footprint ;
	int hitLenRequired ;       // SetHitLenRequired (SeqSet.hpp:2601), 31 by default
	int considerBarcode ;      // SetConsiderBarcodeInIndexHash (SeqSet.hpp:2611)
} ;

#endif
