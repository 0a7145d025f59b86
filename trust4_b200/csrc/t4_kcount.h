// Canonical k-mer counting and per-read count statistics on the device (SURVEY.md 8f-3, the counting part of the
// stage-1 pre-processing):
//
//   KmerCount kmerCount( 21 ) ; kmerCount.AddCount( read ) for every read           KmerCount.hpp:64-97, main.cpp:404-440
//   kmerCount.GetCountStatsAndTrim( read, qual, minCnt, medianCnt, avgCnt )          KmerCount.hpp:177-288, main.cpp:981-1010
//
// (qual == NULL with --trimLevel 0; otherwise the low-quality tail of the read is cut first, KmerCount.hpp:241-271, and
// the statistics cover what is left).  minCnt / medianCnt / avgCnt order the reads
// (main.cpp:103-125) and set the similarity thresholds of the AddRead loop (main.cpp:1675-1694).
//
// The reference keeps 1 000 003 std::maps; here the counts live in one open-addressing table in HBM
// (u64 key = canonical code + 1, u32 count; load factor <= 1/2) filled with one atomicCAS + one atomicAdd per k-mer.
// Both kernels are written against a (lane, group size, group barrier) abstraction: on the GPU a group is a WARP that
// owns a read (persistent warps draw batches of reads from an atomic cursor; no CTA barrier anywhere), in the test-only
// emulation build it is one thread:
//   count  the read becomes one code byte per base in shared memory; a lane owns a contiguous block of positions and
//          rolls the k-mer code and its reverse complement along it (KmerCode::Append; N-free window = IsValid;
//          min of the two = GetCanonicalKmerCode) and inserts every valid k-mer;
//   stats  the same walk with a lookup per k-mer; the counts of the valid k-mers are compacted in position order
//          (scan over the lanes), the median is found by rank counting (the element with exactly m/2 smaller-or-earlier
//          elements is c[m/2] of the sorted array), min and sum by a group reduction; the trimming and the N rules of
//          KmerCount.hpp:241-283 follow.
//
// Per-cell variant (BC = true; the barcode-wise count of --barcode runs, main.cpp:1128-1180): the reference gives every
// barcode group a fresh KmerCount( 21, 23 ) (Clear() between groups), AddCount over the group, then
// GetCountStatsAndTrim( read, NULL, ... ).  Clearing a table per barcode is the same as keying one table by (barcode,
// canonical k-mer): key = code + 1 in the low 43 bits (k <= 21) and barcode - lo above them, so one count launch and one
// statistics launch cover every barcode of [lo, lo + 2^21) in any read order; the host runs one pass per such range that
// holds reads (barcode ids up to 2^31 - 1 stay exact; nothing is hashed into fewer bits).  The slot hash mixes all 64 key
// bits: the global hash only sees the key's low bits, so the same k-mer of many cells would share one probe chain.
// The global pass (BC = false) is the same code with these parts compiled out.
#ifndef T4_KCOUNT_H
#define T4_KCOUNT_H

#include "t4_engine.h"

struct T4KcParams
{
	u64 keys ;             // u64[cap]  (absolute device pointers), 0 = empty, else canonical code + 1
	u64 counts ;           // u32[cap]
	u64 cap ;              // power of two
	u64 pool ;             // ASCII reads
	u64 seqOff ;           // u64[n]
	u64 len ;              // i32[n]
	u64 minCnt, medianCnt ; // i32[n] out
	u64 avgCnt ;           // f32[n] out
	u64 qual ;             // ASCII qualities, same offsets as the reads; 0 = GetCountStatsAndTrim( read, NULL, ... ): no trimming
	u64 newLen ;           // i32[n] out (may be 0): length of the read after the quality trimming
	u64 ctrl ;             // u64[4]: [0] read cursor, [1] k-mers inserted, [2] distinct k-mers, [3] table full flag
	i64 n ;
	int k ;
	int pad ;
} ;

// the barcode of the per-cell pass (a parameter of its own: T4KcParams and the global kernel keep their layout)
struct T4KcBarcode
{
	u64 barcode ;          // i32[n] barcode id of every read
	int lo ;               // this pass counts the reads with lo <= barcode < lo + 2^T4_KC_BC_BITS
	int max ;              // the largest valid barcode id: a read outside [0, max] flags ctrl[3] = 2 (results invalid)
} ;

#define T4_KC_BC_SHIFT 43          /* key bits of code + 1 (k <= 21: code < 2^42) */
#define T4_KC_BC_BITS 21           /* barcode bits of a key: barcode - lo < 2^21 */
#define T4_KC_MAX_POS T4_DEV_MAX_READ
#define T4_KC_MAX_PROBES 4096      /* linear-probe bound: at load <= 1/2 clusters are a few slots long; beyond this the table is treated as full */
#define T4_KC_GROUP 32             /* threads that share a read: one warp (a CTA of 128 per read spent its time at CTA barriers and
                                      the cursor round trip) */
#define T4_KC_BATCH 4              /* reads per cursor step */

struct T4KcSmem                    // per group (warp)
{
	unsigned char code[T4_DEV_MAX_READ + 8] ; // the current read, one byte per base: A 0 C 1 G 2 T 3 (anything else 3, like nucToNum & 3), N 4
	int c[T4_KC_MAX_POS] ;         // counts of the valid k-mers of the current read, compacted in position order
	u32 valid[T4_KC_MAX_POS] ;     // count at position q, 0 = the k-mer at q holds an N
	u32 scan[T4_KC_GROUP + 4] ;
	u64 bu[2] ;
	int bi[8] ;
} ;

T4_HD inline u64 t4_kc_hash( u64 key, u64 cap ) { return ( ( key * 0x9E3779B97F4A7C15ull ) >> 20 ) & ( cap - 1 ) ; }

// per-cell keys: a full 64-bit mix (the splitmix64 finaliser), so that the barcode bits move the slot
T4_HD inline u64 t4_kc_hash_bc( u64 key, u64 cap )
{
	key ^= key >> 33 ;
	key *= 0xFF51AFD7ED558CCDull ;
	key ^= key >> 33 ;
	key *= 0xC4CEB9FE1A85EC53ull ;
	key ^= key >> 33 ;
	return key & ( cap - 1 ) ;
}

// the key bits above the k-mer for read r: false = the read is not counted in this pass (BC only)
template <bool BC> T4_D inline bool kc_read_key( const T4KcParams &P, const T4KcBarcode &B, i64 r, u64 &hi )
{
	hi = 0 ;
	if ( !BC )
		return true ;
	const int b = t4_x<int32_t>( B.barcode )[r] ;
	if ( b < 0 || b > B.max )
	{
		t4_x<u64>( P.ctrl )[3] = 2 ;
		return false ;
	}
	if ( b < B.lo || b - B.lo >= ( 1 << T4_KC_BC_BITS ) )
		return false ;
	hi = (u64)( b - B.lo ) << T4_KC_BC_SHIFT ;
	return true ;
}

// nucToNum[ c - 'A' ] & 3 (main.cpp:39-42) with N kept apart; selects, no branches
T4_HD inline unsigned char t4_kc_code( char c )
{
	return (unsigned char)( c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : c == 'N' ? 4 : 3 ) ;
}

// Rolling KmerCode over the base codes of a read (KmerCode::Append, KmerCode.hpp:94-109) with the canonical code
// (GetCanonicalKmerCode, KmerCode.hpp:52-67: min of the code and its reverse complement) available at every position.
// A thread owns a contiguous block of positions: k - 1 bases of run-in, then one step per position.  The first version
// rebuilt every k-mer from scratch with a branch per character: 60 % of the kernel's instructions (ncu source view).
struct T4KcRoll
{
	u64 fw, rc, mask ;
	int lastN ;                    // position of the last N seen, -1 = none
	int top ;                      // 2 * (k - 1)
} ;

T4_HD inline void t4_kc_roll_start( T4KcRoll &R, const unsigned char *code, int q0, int k )
{
	R.fw = R.rc = 0 ;
	R.mask = k < 32 ? ( ( 1ull << ( 2 * k ) ) - 1ull ) : ~0ull ;
	R.lastN = -1 ;
	R.top = 2 * ( k - 1 ) ;
	for ( int j = 0 ; j < k - 1 ; ++j )
	{
		const unsigned x = code[q0 + j] ;
		if ( x == 4 )
			R.lastN = q0 + j ;
		R.fw = ( R.fw << 2 ) | ( x & 3 ) ;
		R.rc |= (u64)( 3 - ( x & 3 ) ) << ( 2 * ( j + 1 ) ) ; // one slot high: the first step shifts it into place
	}
}

// advance to the k-mer starting at q; false: it holds an N (KmerCode::IsValid)
T4_HD inline bool t4_kc_roll_step( T4KcRoll &R, const unsigned char *code, int q, int k, u64 *canonical )
{
	const unsigned x = code[q + k - 1] ;
	if ( x == 4 )
		R.lastN = q + k - 1 ;
	R.fw = ( ( R.fw << 2 ) | ( x & 3 ) ) & R.mask ;
	R.rc = ( R.rc >> 2 ) | ( (u64)( 3 - ( x & 3 ) ) << R.top ) ;
	*canonical = R.rc < R.fw ? R.rc : R.fw ;
	return R.lastN < q ;
}

struct T4KcCtx
{
	T4KcSmem *sm ;
	int tid, nt ;                  // lane and size of the group that shares a read (a warp; one thread in the emulation)
} ;

#if T4_CUDA
#define T4_KC_SYNC() __syncwarp()
#else
#define T4_KC_SYNC() ((void)0)
#endif

// next batch of reads of this group (atomic cursor): first record, -1 = none left.  Collective.
T4_D inline i64 kc_next_batch( T4KcCtx &cx, const T4KcParams &P )
{
	T4_KC_SYNC() ;
	if ( cx.tid == 0 )
		cx.sm->bu[0] = t4_atomic_add( t4_x<u64>( P.ctrl ), (u64)T4_KC_BATCH ) ;
	T4_KC_SYNC() ;
	const u64 r = cx.sm->bu[0] ;
	T4_KC_SYNC() ;
	return r < (u64)P.n ? (i64)r : -1 ;
}

T4_D inline void kc_load_read( T4KcCtx &cx, const T4KcParams &P, i64 r, int len )
{
	const char *src = t4_x<char>( P.pool ) + t4_x<u64>( P.seqOff )[r] ;
	T4_KC_SYNC() ; // the previous read is done with
	for ( int i = cx.tid ; i < len ; i += cx.nt )
		cx.sm->code[i] = t4_kc_code( src[i] ) ;
	T4_KC_SYNC() ;
}

// KmerCount::AddCount for the reads this group draws (BC: into the table of the read's barcode)
template <bool BC> T4_D inline void kc_count_body( T4KcCtx &cx, const T4KcParams &P, const T4KcBarcode &B )
{
	u64 *keys = t4_x<u64>( P.keys ) ;
	u32 *counts = t4_x<u32>( P.counts ) ;
	u64 *ctrl = t4_x<u64>( P.ctrl ) ;
	u64 inserted = 0, fresh = 0 ;
	for ( i64 r0 = kc_next_batch( cx, P ) ; r0 >= 0 ; r0 = kc_next_batch( cx, P ) )
	for ( i64 r = r0 ; r < r0 + T4_KC_BATCH && r < P.n ; ++r )
	{
		u64 hi ;
		if ( !kc_read_key<BC>( P, B, r, hi ) )
			continue ;
		const int len = t4_x<int32_t>( P.len )[r] ;
		if ( len < P.k || len > T4_DEV_MAX_READ )
			continue ;
		kc_load_read( cx, P, r, len ) ;
		const int m = len - P.k + 1 ;
		const int chunk = ( m + cx.nt - 1 ) / cx.nt ;
		int a = chunk * cx.tid, b = a + chunk ;
		if ( a > m ) a = m ;
		if ( b > m ) b = m ;
		if ( a >= b )
			continue ;
		T4KcRoll R ;
		t4_kc_roll_start( R, cx.sm->code, a, P.k ) ;
		for ( int q = a ; q < b ; ++q )
		{
			u64 code ;
			if ( !t4_kc_roll_step( R, cx.sm->code, q, P.k, &code ) )
				continue ;
			const u64 key = BC ? ( code + 1 ) | hi : code + 1 ;
			u64 s = BC ? t4_kc_hash_bc( key, P.cap ) : t4_kc_hash( key, P.cap ) ;
			u64 probes = 0 ;
			while ( 1 )
			{
				u64 cur = keys[s] ;
				if ( cur == 0 )
				{
					cur = t4_atomic_cas( keys + s, 0ull, key ) ;
					if ( cur == 0 )
					{
						cur = key ;
						++fresh ;
					}
				}
				if ( cur == key )
				{
					t4_atomic_add32( counts + s, 1u ) ;
					++inserted ;
					break ;
				}
				s = ( s + 1 ) & ( P.cap - 1 ) ;
				if ( ++probes > T4_KC_MAX_PROBES )
				{
					ctrl[3] = 1 ; // table (nearly) full: the caller's capacity hint was too small; the results are flagged invalid
					break ;
				}
			}
		}
	}
	if ( inserted )
		t4_atomic_add( ctrl + 1, inserted ) ;
	if ( fresh )
		t4_atomic_add( ctrl + 2, fresh ) ;
}

template <bool BC> T4_D inline u32 kc_lookup( const T4KcParams &P, u64 code, u64 hi )
{
	const u64 *keys = t4_x<u64>( P.keys ) ;
	const u64 key = BC ? ( code + 1 ) | hi : code + 1 ;
	u64 s = BC ? t4_kc_hash_bc( key, P.cap ) : t4_kc_hash( key, P.cap ) ;
	for ( int probes = 0 ; probes <= T4_KC_MAX_PROBES ; ++probes ) // bounded like the insert: an overfull table cannot hang the launch
	{
		const u64 cur = keys[s] ;
		if ( cur == key )
			return t4_x<u32>( P.counts )[s] ;
		if ( cur == 0 )
			return 0 ;
		s = ( s + 1 ) & ( P.cap - 1 ) ;
	}
	return 0 ;
}

// exclusive scan of one value per thread + total (same contract as the engine's c_scan_threads, on T4KcSmem)
T4_D inline u32 kc_scan( T4KcCtx &cx, u32 v, u32 &total )
{
	T4_KC_SYNC() ;
	cx.sm->scan[cx.tid] = v ;
	T4_KC_SYNC() ;
	u32 base = 0, tot = 0 ;
	for ( int t = 0 ; t < cx.nt ; ++t )
	{
		const u32 x = cx.sm->scan[t] ;
		if ( t < cx.tid )
			base += x ;
		tot += x ;
	}
	total = tot ;
	T4_KC_SYNC() ;
	return base ;
}

// KmerCount::GetCountStatsAndTrim( read, qual, ... ) for the reads this group draws (BC: qual is 0; the reads of other
// passes are left alone)
template <bool BC> T4_D inline void kc_stats_body( T4KcCtx &cx, const T4KcParams &P, const T4KcBarcode &B )
{
	T4KcSmem *sm = cx.sm ;
	int32_t *minCnt = t4_x<int32_t>( P.minCnt ), *medianCnt = t4_x<int32_t>( P.medianCnt ) ;
	float *avgCnt = t4_x<float>( P.avgCnt ) ;
	for ( i64 r0 = kc_next_batch( cx, P ) ; r0 >= 0 ; r0 = kc_next_batch( cx, P ) )
	for ( i64 r = r0 ; r < r0 + T4_KC_BATCH && r < P.n ; ++r )
	{
		u64 hi ;
		if ( !kc_read_key<BC>( P, B, r, hi ) )
			continue ;
		const int len = t4_x<int32_t>( P.len )[r] ;
		if ( len < P.k || len > T4_DEV_MAX_READ )
		{
			if ( cx.tid == 0 )
			{
				minCnt[r] = medianCnt[r] = -1 ; // KmerCount.hpp:196-200 (longer than the device limit: not supported, flagged by the host)
				avgCnt[r] = -1.0f ;
				if ( P.newLen )
					t4_x<int32_t>( P.newLen )[r] = len ;
			}
			continue ;
		}
		kc_load_read( cx, P, r, len ) ;
		const int m = len - P.k + 1 ;
		// counts of the valid k-mers, compacted in position order (the reference's c[0..k))
		// pass 1: validity + count per position (a thread owns a contiguous block of positions so the compaction is a scan)
		const int chunk = ( m + cx.nt - 1 ) / cx.nt ;
		int a = chunk * cx.tid, b = a + chunk ;
		if ( a > m ) a = m ;
		if ( b > m ) b = m ;
		u32 nv = 0 ;
		T4KcRoll R ;
		if ( a < b )
			t4_kc_roll_start( R, sm->code, a, P.k ) ;
		for ( int q = a ; q < b ; ++q )
		{
			u64 code ;
			if ( t4_kc_roll_step( R, sm->code, q, P.k, &code ) )
			{
				int c = (int)kc_lookup<BC>( P, code, hi ) ;
				if ( c <= 0 )
					c = 1 ; // KmerCount.hpp:222-223
				sm->valid[q] = (u32)c ;
				++nv ;
			}
			else
				sm->valid[q] = 0 ;
		}
		u32 total ;
		u32 o = kc_scan( cx, nv, total ) ;
		for ( int q = a ; q < b ; ++q )
			if ( sm->valid[q] )
				sm->c[o++] = (int)sm->valid[q] ;
		T4_KC_SYNC() ;
		const int kk = (int)total ;
		int32_t *newLen = t4_x<int32_t>( P.newLen ) ;
		if ( kk == 0 )
		{
			if ( cx.tid == 0 )
			{
				minCnt[r] = medianCnt[r] = -len ; // KmerCount.hpp:229-239
				avgCnt[r] = (float)( -len ) ;
				if ( newLen )
					newLen[r] = P.qual ? 0 : len ; // `if ( qual != NULL ) read[0] = '\0'`
			}
			continue ;
		}
		// quality trimming (KmerCount.hpp:241-271), serial: the tail behind the last k-mer seen more than once is scanned from
		// the end; the read is cut at the leftmost position where the bad bases (Phred <= 15) reach 10 % of the tail
		int kUse = kk, trimStart = -1 ;
		if ( P.qual )
		{
			if ( cx.tid == 0 )
			{
				const char *q = t4_x<char>( P.qual ) + t4_x<u64>( P.seqOff )[r] ;
				int i ;
				for ( i = kk - 1 ; i >= 0 ; --i )
					if ( sm->c[i] > 1 )
						break ;
				++i ;
				int badCnt = 0, ts = -1 ;
				for ( int j = len - 1 ; j >= i + P.k - 1 ; --j )
					if ( q[j] - 32 <= 15 )
					{
						++badCnt ;
						if ( badCnt >= 0.1 * ( len - j ) )
							ts = j ;
					}
				int ku = kk ;
				if ( ts > 0 )
					ku = ts - P.k + 1 ;
				if ( ts > 0 && ts < P.k )
					ku = 0 ;
				if ( ku > kk )
					ku = kk ; // only with N's in a trimmed read: the reference then sorts stale entries of its shared buffer (undefined)
				sm->bi[2] = ku ;
				sm->bi[3] = ts ;
			}
			T4_KC_SYNC() ;
			kUse = sm->bi[2] ;
			trimStart = sm->bi[3] ;
			T4_KC_SYNC() ;
		}
		// min and the element of sorted rank kUse / 2 over the first kUse counts; the sum runs over ALL counts (the reference
		// sums before it trims, KmerCount.hpp:224, 274)
		int mn = 0x7fffffff ;
		u32 sum = 0 ;
		int med = -1 ;
		for ( int i = cx.tid ; i < kk ; i += cx.nt )
		{
			const int v = sm->c[i] ;
			sum += (u32)v ;
			if ( i >= kUse )
				continue ;
			if ( v < mn )
				mn = v ;
			int rank = 0 ;
			for ( int j = 0 ; j < kUse ; ++j )
			{
				const int w = sm->c[j] ;
				if ( w < v || ( w == v && j < i ) )
					++rank ;
			}
			if ( rank == kUse / 2 )
				med = v ;
		}
		// CTA reductions through shared memory (one slot per thread)
		T4_KC_SYNC() ;
		sm->scan[cx.tid] = (u32)mn ;
		T4_KC_SYNC() ;
		if ( cx.tid == 0 )
		{
			int x = 0x7fffffff ;
			for ( int t = 0 ; t < cx.nt ; ++t )
				if ( (int)sm->scan[t] < x )
					x = (int)sm->scan[t] ;
			sm->bi[0] = x ;
		}
		T4_KC_SYNC() ;
		u32 sumTotal ;
		kc_scan( cx, sum, sumTotal ) ;
		if ( med >= 0 )
			sm->bi[1] = med ; // exactly one thread holds the rank kUse / 2 element
		T4_KC_SYNC() ;
		if ( cx.tid == 0 )
		{
			const bool dropped = trimStart > 0 && trimStart < P.k ; // read[0] = '\0': the driver discards the read
			int minCount = kUse > 0 ? sm->bi[0] : sm->c[0] ;          // std::sort over nothing: c[0] is the first count as it stands
			const int medianCount = kUse > 0 ? sm->bi[1] : sm->c[0] ;
			for ( int i = 0 ; i < len ; ++i ) // KmerCount.hpp:275-283: over the ORIGINAL length; the cut only overwrote read[trimStart] (and read[0])
			{
				if ( ( trimStart > 0 && i == trimStart ) || ( dropped && i == 0 ) )
					continue ;
				if ( sm->code[i] == 4 )
				{
					if ( minCount >= 0 )
						minCount = 0 ;
					else if ( minCount <= 0 )
						--minCount ;
				}
			}
			minCnt[r] = minCount ;
			medianCnt[r] = medianCount ;
			avgCnt[r] = (float)( (int)sumTotal / (double)kUse ) ; // `avgCount = sum / (double)k` into a float, KmerCount.hpp:274 (k = 0: inf)
			if ( newLen )
				newLen[r] = trimStart > 0 ? ( dropped ? 0 : trimStart ) : len ;
		}
	}
}

#endif
