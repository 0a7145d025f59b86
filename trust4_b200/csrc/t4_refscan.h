// Stage-0 candidate extraction on the device (SURVEY.md 8f-4): the per-read predicate of `fastq-extractor`
//
//   IsGoodCandidate( read ) = !IsLowComplexity( read ) && refSet->HasHitInSet( read, 0 ) != 0      FastqExtractor.cpp:106-134
//   int SeqSet::HasHitInSet( char *read, int mode )                                                 SeqSet.hpp:3144-3327
//
// against the reference gene set (`SeqSet refSet( 9 ) ; refSet.InputRefFa( file )`, FastqExtractor.cpp:316-318): seed hits
// of both strands (GetHitsFromRead), the hits bucketed per (strand, gene), the bucket with the most distinct read
// positions per strand, and GetOverlapsFromHits on the winning bucket(s) -- for REFERENCE sequences, i.e. the branch of
// SeqSet.hpp:763-1063 the assembly path never takes: diagonal windows of radius 10, a longest increasing subsequence with
// the reference's tie rules, hit lengths on read and gene.
//
// It is the volume scan of the pipeline (every raw read, typically 1e8) and read-only, so it runs like the AssignRead
// pass: worker CTAs of the auxiliary kernel over the whole GPU, reads from an atomic cursor.  The probe and the key sort
// are the engine's collectives; the bucket statistics and the chain logic are serial per read (a few hundred hits) and
// plain C, identical on the device and in the test emulation.
#ifndef T4_REFSCAN_H
#define T4_REFSCAN_H

#include "t4_assign.h"

struct T4RefInput          // T4_OP_REF_INPUT: sequences to append to the set (device buffers, absolute pointers)
{
	u64 seqPool ;          // char[]: sequences back to back
	u64 seqOff ;           // u64[n + 1]
	u64 namePool ;         // char[]
	u64 nameOff ;          // u64[n + 1]
	int n ;
	int pad ;
} ;

struct T4ScanParams        // T4_OP_REF_SCAN
{
	u64 pool ;             // ASCII reads
	u64 seqOff ;           // u64[n]
	u64 len ;              // i32[n]
	u64 strandOut ;        // i8[n]: HasHitInSet( read, 0 ): 0 no hit, +1 / -1 strand
	u64 lowOut ;           // u8[n]: IsLowComplexity( read )
	u64 cursor ;           // u64[4]: [0] read cursor, [1] reads with a hit, [2] low-complexity reads
	u64 setOff ;           // arena offset of the reference set's stream
	i64 n ;
} ;

#define T4_SCAN_CHUNK 8

// ---- InputRefFa, device part: one contig per (cleaned, de-duplicated) sequence, indexed like any contig -----------------
// (SeqSet.hpp:2707-2712, 2864: seqIndex.BuildIndexFromRead( kmerCode, consensus, len, id, -1 ))
T4_D inline void c_ref_input( T4Ctx &cx, T4Op *op )
{
	const T4RefInput *in = t4_x<T4RefInput>( op->out ) ;
	T4Smem *sm = cx.sm ;
	const u64 *seqOff = t4_x<u64>( in->seqOff ), *nameOff = t4_x<u64>( in->nameOff ) ;
	for ( int s = 0 ; s < in->n ; ++s )
	{
		const int len = (int)( seqOff[s + 1] - seqOff[s] ) ;
		const char *src = t4_x<char>( in->seqPool ) + seqOff[s] ;
		T4_SYNC() ;
		if ( cx.tid == 0 )
		{
			s_refill_slab( cx ) ;
			int idx = s_new_contig( cx, len ) ;
			if ( idx >= 0 )
			{
				T4Contig *c = t4_seq( cx, idx ) ;
				s_set_name( cx, c, t4_x<char>( in->namePool ) + nameOff[s], (int)( nameOff[s + 1] - nameOff[s] ) ) ;
				c->barcode = -1 ;
				c->numRead = 0 ;
			}
			sm->bi[0] = idx ;
		}
		T4_SYNC() ;
		const int idx = sm->bi[0] ;
		T4_SYNC() ;
		if ( idx < 0 || c_uniform_error( cx ) )
			break ;
		T4Contig *c = t4_seq( cx, idx ) ;
		char *cons = t4_cons( cx, c ) ;
		int *pw = t4_pw( cx, c ) ;
		unsigned char *eq = t4_eq( cx, c ) ;
		T4_PAR_FOR( i, len )
		{
			cons[i] = src[i] ;
			t4_col_put( pw, eq, i, 0, 0, 0, 0 ) ;
		}
		T4_SYNC() ;
		c_index_op( cx, cons, len, T4_IDX_BUILD, idx, -1, 0, 0 ) ;
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
		op->ret = cx.st->error ? cx.st->error : cx.st->nSeqs ;
}

// ---- serial helpers (thread 0) ------------------------------------------------------------------------------------
T4_HD inline void t4_heapsort64( u64 *a, int n )
{
	for ( int start = n / 2 - 1 ; start >= 0 ; --start )
	{
		int root = start ;
		while ( 2 * root + 1 < n )
		{
			int child = 2 * root + 1 ;
			if ( child + 1 < n && a[child] < a[child + 1] )
				++child ;
			if ( a[root] >= a[child] )
				break ;
			u64 t = a[root] ; a[root] = a[child] ; a[child] = t ;
			root = child ;
		}
	}
	for ( int end = n - 1 ; end > 0 ; --end )
	{
		u64 t = a[0] ; a[0] = a[end] ; a[end] = t ;
		int root = 0 ;
		while ( 2 * root + 1 < end )
		{
			int child = 2 * root + 1 ;
			if ( child + 1 < end && a[child] < a[child + 1] )
				++child ;
			if ( a[root] >= a[child] )
				break ;
			u64 t2 = a[root] ; a[root] = a[child] ; a[child] = t2 ;
			root = child ;
		}
	}
}

T4_HD inline double t4_absd( double x ) { return x < 0 ? -x : x ; }

// SeqSet::BinarySearch_LIS, SeqSet.hpp:316-337
T4_HD inline int t4_lis_search( const int *top, int size, int valA, const int *ha )
{
	int l = 0, r = size - 1 ;
	while ( l <= r )
	{
		int m = ( l + r ) / 2 ;
		if ( valA == ha[ top[m] ] )
			return m ;
		else if ( valA < ha[ top[m] ] )
			r = m - 1 ;
		else
			l = m + 1 ;
	}
	return l - 1 ;
}

// SeqSet::LongestIncreasingSubsequence, SeqSet.hpp:342-474: hits (ha, hb), sorted by b; the subsequence (increasing in a,
// one element per b, the least divergent from the average diagonal on ties, then the replacement sweep) goes to (oa, ob).
// top / link: scratch of `size` ints each.  Returns its length.
T4_HD inline int t4_lis( const int *ha, const int *hb, int size, int *top, int *link, int *oa, int *ob )
{
	double avgDiff = 0 ;
	for ( int i = 1 ; i < size ; ++i )
		avgDiff += ( ha[i] - hb[i] ) ;
	avgDiff /= size ;
	top[0] = 0 ;
	link[0] = -1 ;
	int ret = 1 ;
	for ( int i = 1 ; i < size ; ++i )
	{
		int tag ;
		if ( ha[ top[ret - 1] ] <= ha[i] )
			tag = ret - 1 ;
		else
			tag = t4_lis_search( top, ret, ha[i], ha ) ;
		if ( tag == -1 )
		{
			top[0] = i ;
			link[i] = -1 ;
		}
		else if ( ha[i] > ha[ top[tag] ] )
		{
			if ( tag == ret - 1 )
			{
				top[ret] = i ;
				++ret ;
				link[i] = top[tag] ;
			}
			else if ( ha[i] < ha[ top[tag + 1] ] )
			{
				top[tag + 1] = i ;
				link[i] = top[tag] ;
			}
		}
		else if ( ha[i] == ha[ top[tag] ] ) // repeats
		{
			if ( t4_absd( ha[i] - hb[i] - avgDiff ) < t4_absd( ha[ top[tag] ] - hb[ top[tag] ] - avgDiff ) )
			{
				top[tag] = i ;
				link[i] = tag > 0 ? top[tag - 1] : -1 ;
			}
		}
	}
	int k = top[ret - 1] ;
	for ( int i = ret - 1 ; i >= 0 ; --i )
	{
		oa[i] = ha[k] ;
		ob[i] = hb[k] ;
		k = link[k] ;
	}
	// one element per b: the least divergent
	{
		int kk = 0 ;
		for ( int i = 0 ; i < ret ; )
		{
			int j ;
			for ( j = i + 1 ; j < ret ; ++j )
				if ( ob[i] != ob[j] )
					break ;
			int mintag = i ;
			if ( j != i + 1 )
			{
				double minDiff = t4_absd( oa[i] - ob[i] - avgDiff ) ;
				for ( int l = i + 1 ; l < j ; ++l )
					if ( t4_absd( oa[l] - ob[l] - avgDiff ) < minDiff )
					{
						minDiff = t4_absd( oa[l] - ob[l] - avgDiff ) ;
						mintag = l ;
					}
			}
			oa[kk] = oa[mintag] ;
			ob[kk] = ob[mintag] ;
			i = j ;
			++kk ;
		}
		ret = kk ;
	}
	// replacement sweep: a hit between two chain elements that fits and lies closer to the average diagonal takes the place
	{
		int i = 0, j = 0 ;
		while ( i < ret && j < size )
		{
			if ( hb[j] < ob[i] )
				++j ;
			else if ( i + 1 < ret && ob[i + 1] <= hb[j] )
				++i ;
			else if ( oa[i] == ha[j] && ob[i] == hb[j] )
				++j ;
			else
			{
				if ( oa[i] <= ha[j] && ( i == ret - 1 || ha[j] < oa[i + 1] )
					&& t4_absd( ha[j] - hb[j] - avgDiff ) < t4_absd( oa[i] - ob[i] - avgDiff ) )
				{
					oa[i] = ha[j] ;
					ob[i] = hb[j] ;
				}
				++j ;
			}
		}
	}
	return ret ;
}

// SeqSet::GetTotalHitLengthOnRead / OnSeq, SeqSet.hpp:476-513, over one coordinate of the chain
T4_HD inline int t4_total_hit_length( const int *x, int n, int k )
{
	int ret = 0 ;
	for ( int i = 0 ; i < n ; )
	{
		int j ;
		for ( j = i + 1 ; j < n ; ++j )
			if ( x[j] > x[j - 1] + k - 1 )
				break ;
		ret += x[j - 1] - x[i] + k ;
		i = j ;
	}
	return ret ;
}

struct T4ScanScratch       // serial work arrays of one worker, each with room for every hit of a read
{
	u64 *w ;               // packed (diagonal, b, a) of the bucket, then (b, a) of a window
	int *ha, *hb, *top, *link, *oa, *ob ;
} ;

// SeqSet::GetOverlapsFromHits( bucket, hitLenRequired, filter = 1, conservativeChain = false ) for ONE bucket of hits on a
// reference sequence (SeqSet.hpp:763-1063, the isRef branch; every posting list of a reference set is far below the 10000
// entries of the `repeats` rules, the caller checks).  keys[0..n): the bucket's hits, re-keyed (a in bits 30.., b in bits
// 1..).  Returns matchCnt of the first overlap the reference would produce, or -1 when it produces none.
T4_HD inline int t4_ref_bucket_overlap( const u64 *keys, int n, int k, int radius, int hitLenRequired, T4ScanScratch &S )
{
	const int minHitRequired = 3 ; // refMinHitRequired, SeqSet.hpp:778, 835-836
	if ( n < minHitRequired )
		return -1 ;
	for ( int i = 0 ; i < n ; ++i )
	{
		const int a = (int)( ( keys[i] >> 30 ) & 0x7ff ), b = (int)( ( keys[i] >> 1 ) & T4_KEY_B_MASK ) ;
		S.w[i] = ( (u64)( a - b + T4_KEY_C_BIAS ) << 40 ) | ( (u64)b << 20 ) | (u64)a ; // CompSortHitCoordDiff: c, then b, then a
	}
	t4_heapsort64( S.w, n ) ;
	for ( int s = 0 ; s < n ; )
	{
		int e ;
		for ( e = s + 1 ; e < n ; ++e )
		{
			int diff = (int)( S.w[e] >> 40 ) - (int)( S.w[e - 1] >> 40 ) ;
			if ( diff < 0 )
				diff = -diff ;
			if ( diff > radius )
				break ;
		}
		if ( e - s < minHitRequired || ( e - s ) * k < hitLenRequired )
		{
			s = e ;
			continue ;
		}
		const int m = e - s ;
		// concordant hits, sorted by b (then a) when the window spans several diagonals (SeqSet.hpp:957-958)
		u64 *cw = S.w + n ;
		for ( int x = 0 ; x < m ; ++x )
			cw[x] = S.w[s + x] & ( ( 1ull << 40 ) - 1ull ) ; // b << 20 | a
		if ( radius > 0 )
			t4_heapsort64( cw, m ) ;
		for ( int x = 0 ; x < m ; ++x )
		{
			S.ha[x] = (int)( cw[x] & 0xfffff ) ;
			S.hb[x] = (int)( cw[x] >> 20 ) ;
		}
		int lisSize = t4_lis( S.ha, S.hb, m, S.top, S.link, S.oa, S.ob ) ;
		if ( lisSize * k < hitLenRequired )
		{
			s = e ;
			continue ;
		}
		const int hitLen = t4_total_hit_length( S.oa, lisSize, k ) ;
		if ( hitLen < hitLenRequired || t4_total_hit_length( S.ob, lisSize, k ) < hitLenRequired )
		{
			s = e ;
			continue ;
		}
		return 2 * hitLen ; // no.matchCnt, SeqSet.hpp:1037
	}
	return -1 ;
}

// The decision of HasHitInSet( read, 0 ) from the read's hits sorted by (strand, gene, read offset, gene offset).
T4_HD inline int t4_has_hit_decide( const u64 *keys, int H, int k, int radius, int hitLenRequired, T4ScanScratch &S )
{
	int max[2] = { -1, -1 }, start[2] = { 0, 0 }, size[2] = { 0, 0 } ;
	for ( int i = 0 ; i < H ; )
	{
		const u64 g = keys[i] >> T4_KEY_IDX_SHIFT ; // strand | gene
		int j = i + 1, readHitCount = 1 ;
		for ( ; j < H && ( keys[j] >> T4_KEY_IDX_SHIFT ) == g ; ++j )
			if ( ( ( keys[j] >> 30 ) & 0x7ff ) != ( ( keys[j - 1] >> 30 ) & 0x7ff ) )
				++readHitCount ;
		const int tag = ( keys[i] >> T4_KEY_STRAND_SHIFT ) ? 1 : 0 ;
		if ( readHitCount > max[tag] ) // genes in ascending order: the first of equals stays (SeqSet.hpp:3184-3188)
		{
			max[tag] = readHitCount ;
			start[tag] = i ;
			size[tag] = j - i ;
		}
		i = j ;
	}
	int maxTag, found ;
	if ( max[0] + k - 1 >= hitLenRequired && max[1] + k - 1 >= hitLenRequired )
	{
		// both strands look good: the better chain decides (SeqSet.hpp:3264-3301)
		const int m0 = t4_ref_bucket_overlap( keys + start[0], size[0], k, radius, hitLenRequired, S ) ;
		const int m1 = t4_ref_bucket_overlap( keys + start[1], size[1], k, radius, hitLenRequired, S ) ;
		if ( m0 >= 0 && m1 >= 0 )
			maxTag = m0 >= m1 ? 0 : 1 ;
		else if ( m0 >= 0 )
			maxTag = 0 ;
		else
			maxTag = 1 ;
		found = maxTag == 0 ? m0 >= 0 : m1 >= 0 ;
	}
	else
	{
		maxTag = max[1] >= max[0] ? 1 : 0 ;
		found = t4_ref_bucket_overlap( keys + start[maxTag], size[maxTag], k, radius, hitLenRequired, S ) >= 0 ;
	}
	if ( !found )
		return 0 ;
	return maxTag == 0 ? -1 : 1 ;
}

// IsLowComplexity, FastqExtractor.cpp:106-127
T4_HD inline int t4_low_complexity_read( const char *seq, int len )
{
	int cnt[5] = { 0, 0, 0, 0, 0 } ;
	for ( int i = 0 ; i < len ; ++i )
	{
		if ( seq[i] == 'N' )
			++cnt[4] ;
		else
			++cnt[ t4_nuc( seq[i] ) ] ;
	}
	const int i = len ;
	if ( cnt[0] >= i / 2 || cnt[1] >= i / 2 || cnt[2] >= i / 2 || cnt[3] >= i / 2 || cnt[4] >= i / 10 )
		return 1 ;
	int lowCnt = 0 ;
	for ( int x = 0 ; x < 4 ; ++x )
		if ( cnt[x] <= 2 )
			++lowCnt ;
	return lowCnt >= 2 ? 1 : 0 ;
}

// ---- T4_OP_REF_SCAN: worker loop -------------------------------------------------------------------------------------
T4_D inline void c_ref_scan( T4Ctx &cx, T4Op *op )
{
	const T4ScanParams *P = t4_x<T4ScanParams>( op->out ) ;
	T4Smem *sm = cx.sm ;
	T4Stream *st = cx.st ;
	const u64 *seqOff = t4_x<u64>( P->seqOff ) ;
	const int32_t *lens = t4_x<int32_t>( P->len ) ;
	const char *pool = t4_x<char>( P->pool ) ;
	int8_t *strandOut = t4_x<int8_t>( P->strandOut ) ;
	unsigned char *lowOut = t4_x<unsigned char>( P->lowOut ) ;
	u64 *cursor = t4_x<u64>( P->cursor ) ;
	c_assign_attach( cx, cx.P<T4Stream>( P->setOff ) ) ;
	u64 nHit = 0, nLow = 0 ;
	bool failed = false ;
	while ( !failed )
	{
		T4_SYNC() ;
		if ( cx.tid == 0 )
			sm->bu[0] = t4_atomic_add( cursor, (u64)T4_SCAN_CHUNK ) ;
		T4_SYNC() ;
		const i64 c0 = (i64)sm->bu[0] ;
		if ( c0 >= P->n )
			break ;
		const i64 c1 = c0 + T4_SCAN_CHUNK < P->n ? c0 + T4_SCAN_CHUNK : P->n ;
		for ( i64 r = c0 ; r < c1 ; ++r )
		{
			const int len = lens[r] ;
			if ( len > T4_DEV_MAX_READ )
			{
				if ( cx.tid == 0 )
				{
					strandOut[r] = 0 ;
					lowOut[r] = 0 ;
					t4_raise( cx, T4_E_UNSUPPORTED, 5 ) ;
				}
				failed = c_uniform_error( cx ) != 0 ;
				break ;
			}
			c_load_read( cx, pool + seqOff[r], len ) ;
			int result = 0 ;
			if ( len >= st->kmerLength )
			{
				int anyBig = 0 ;
				u32 H = c_get_hits( cx, len, 0, -1, false, &anyBig, true ) ;
				if ( anyBig && cx.tid == 0 )
					t4_raise( cx, T4_E_UNSUPPORTED, 6 ) ; // a k-mer with > 10000 postings: not a reference gene set
				failed = c_uniform_error( cx ) != 0 ;
				if ( failed )
					break ;
				if ( H > 0 )
				{
					// SortHits order (strand, gene, read offset, gene offset): buckets become ranges
					u64 *a = cx.P<u64>( st->keysAOff ) ;
					u64 *b = cx.P<u64>( st->keysBOff ) ;
					T4_PAR_FOR( i, H )
					{
						const u64 kx = a[i] ;
						a[i] = ( kx & ( ~0ull << T4_KEY_IDX_SHIFT ) ) | ( (u64)t4_key_a( kx ) << 30 ) | ( (u64)t4_key_b( kx ) << 1 ) | ( kx & 1 ) ;
					}
					T4_SYNC() ;
					u64 *sorted = c_sort_keys( cx, a, b, H ) ;
					u64 *tmp = ( sorted == a ) ? b : a ;
					// serial work arrays: 2 H packed words in the free key buffer (grown with the hit buffers: hitCap >= H, and
					// the bucket and its window never exceed H together only when split -- so a second area holds the window)
					T4_SYNC() ;
					const u32 capR = st->hitCapR ; // read by everybody BEFORE thread 0 may change it: the branch below holds barriers
					T4_SYNC() ;
					if ( 2 * H > capR )
					{
						if ( cx.tid == 0 )
						{
							u32 nc = capR ? capR : 4096 ;
							while ( nc < 2 * H )
								nc *= 2 ;
							u64 x = s_alloc( cx, (u64)nc * 8 ) ;
							u64 y = s_alloc( cx, (u64)nc * 8 ) ;
							if ( x && y )
							{
								st->keysROff = x ;
								st->keysR2Off = y ;
								st->hitCapR = nc ;
							}
						}
						failed = c_uniform_error( cx ) != 0 ;
						if ( failed )
							break ;
					}
					if ( cx.tid == 0 )
					{
						T4ScanScratch S ;
						S.w = cx.P<u64>( st->keysROff ) ;                 // 2 H words: bucket, then window
						int *ia = (int *)cx.P<u64>( st->keysR2Off ) ;     // 4 H ints
						S.ha = ia ; S.hb = ia + H ; S.top = ia + 2 * H ; S.link = ia + 3 * H ;
						S.oa = (int *)tmp ; S.ob = (int *)tmp + H ;        // 2 H ints in the free key buffer (H words)
						result = t4_has_hit_decide( sorted, (int)H, st->kmerLength, st->radius, st->hitLenRequired, S ) ;
					}
				}
			}
			if ( cx.tid == 0 )
			{
				const int low = t4_low_complexity_read( sm->read, len ) ;
				strandOut[r] = (int8_t)result ;
				lowOut[r] = (unsigned char)low ;
				if ( result != 0 )
					++nHit ;
				if ( low )
					++nLow ;
			}
		}
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
	{
		if ( nHit )
			t4_atomic_add( cursor + 1, nHit ) ;
		if ( nLow )
			t4_atomic_add( cursor + 2, nLow ) ;
		op->ret = cx.st->error ? cx.st->error : 0 ;
	}
}

T4_D inline void c_run_aux_op_more( T4Ctx &cx, T4Op *op )
{
	switch ( op->op )
	{
		case T4_OP_REF_INPUT:
			c_ref_input( cx, op ) ;
			break ;
		case T4_OP_REF_SCAN:
			c_ref_scan( cx, op ) ;
			break ;
		default:
			break ;
	}
}

#endif
