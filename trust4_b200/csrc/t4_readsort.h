// The read order of the stage-1 driver on the device (SURVEY.md 8f-3: "the sort"): `std::sort( sortedReads )` with
// `_sortRead::operator<` (main.cpp:103-125, 1078) -- minCnt, medianCnt, avgCnt and length descending, then the read
// string and the id ascending.  The order decides what the serial AddRead loop sees first, so it has to be exact; the
// comparator is a strict total order on distinct records, hence any correct sort yields the reference's sequence.
//
// A bottom-up merge sort over an index array: in the pass of run width w every element finds its place among the 2w
// elements of its pair of runs by ONE binary search in the partner run (lower bound for the left run's elements, upper
// bound for the right run's: stable) -- n independent searches per pass, log2 n passes, no shared state.
//
// STATUS: verified on an H100 (tests/test_gpu_preprocess.py) against the reference's std::sort and, at 2^20 + 3 records
// (more than one grid of the grid-stride loop), against a Python restatement of the comparator; a kernel of its own
// (t4_readsort_kernel).  The --barcode order (CompReadWithBarcode, T4SortRecBc below) is the same merge body over a wider
// record (t4_readsort_bc_kernel), verified the same way (tests/test_gpu_barcode_stats.py).
#ifndef T4_READSORT_H
#define T4_READSORT_H

#include "t4_common.h"

struct T4SortRec           // what _sortRead::operator< looks at
{
	int32_t minCnt, medianCnt ;
	float avgCnt ;
	int32_t len ;          // strlen( read )
	u64 readOff ;          // into the read pool
	u64 idOff ;            // into the id pool
	int32_t idLen ;
	int32_t pad ;
} ;

struct T4SortParams
{
	u64 recs ;             // T4SortRec[n]       (absolute device pointers)
	u64 pool, idPool ;
	u64 src, dst ;         // i64[n] index arrays of this pass
	i64 n ;
	i64 width ;            // run length of the pass
} ;

// strcmp on a (pointer, length) pair: bytes as unsigned char, the shorter string first on a common prefix
T4_HD inline int t4_strcmp_n( const char *a, int la, const char *b, int lb )
{
	const int m = la < lb ? la : lb ;
	for ( int i = 0 ; i < m ; ++i )
	{
		const unsigned char x = (unsigned char)a[i], y = (unsigned char)b[i] ;
		if ( x != y )
			return x < y ? -1 : 1 ;
	}
	return la == lb ? 0 : ( la < lb ? -1 : 1 ) ;
}

// _sortRead::operator<, main.cpp:103-125
T4_HD inline bool t4_sortrec_less( const T4SortRec &a, const T4SortRec &b, const char *pool, const char *idPool )
{
	if ( a.minCnt != b.minCnt )
		return a.minCnt > b.minCnt ;
	else if ( a.medianCnt != b.medianCnt )
		return a.medianCnt > b.medianCnt ;
	else if ( a.avgCnt != b.avgCnt )
		return a.avgCnt > b.avgCnt ;
	else if ( a.len != b.len )
		return a.len > b.len ;
	const int tmp = t4_strcmp_n( pool + a.readOff, a.len, pool + b.readOff, b.len ) ;
	if ( tmp != 0 )
		return tmp < 0 ;
	return t4_strcmp_n( idPool + a.idOff, a.idLen, idPool + b.idOff, b.idLen ) < 0 ;
}

// The record of the --barcode order: `CompReadWithBarcode` (main.cpp:128-136) -- barcode ascending, barcodeMinCnt
// descending, then _sortRead::operator<.  A record of its own, so that the global sort keeps its record and its kernel.
// The reference's comparator special-cases barcode -1 and is a strict weak order only when every barcode is >= 0 (with
// --barcode every read has one, main.cpp:797-819); the entry point rejects negative barcodes, and for barcodes >= 0 the
// comparison below is the reference's.
struct T4SortRecBc
{
	T4SortRec r ;
	int32_t barcode, barcodeMinCnt ;
} ;

T4_HD inline bool t4_sortrec_less( const T4SortRecBc &a, const T4SortRecBc &b, const char *pool, const char *idPool )
{
	if ( a.barcode != b.barcode )
		return a.barcode < b.barcode ;
	else if ( a.barcodeMinCnt != b.barcodeMinCnt )
		return a.barcodeMinCnt > b.barcodeMinCnt ;
	return t4_sortrec_less( a.r, b.r, pool, idPool ) ;
}

// output position of src[i] in the merge of its pair of runs (Rec: T4SortRec or T4SortRecBc)
template <class Rec> T4_HD inline void t4_sort_merge_one( const T4SortParams &P, i64 i )
{
	const Rec *recs = t4_x<Rec>( P.recs ) ;
	const char *pool = t4_x<char>( P.pool ), *idPool = t4_x<char>( P.idPool ) ;
	const i64 *src = t4_x<i64>( P.src ) ;
	i64 *dst = t4_x<i64>( P.dst ) ;
	const i64 w = P.width ;
	const i64 base = ( i / ( 2 * w ) ) * ( 2 * w ) ;
	const i64 aEnd = base + w < P.n ? base + w : P.n ;
	const i64 bEnd = base + 2 * w < P.n ? base + 2 * w : P.n ;
	const Rec &x = recs[ src[i] ] ;
	if ( i < aEnd )
	{
		// left run: count the right run's elements that come strictly before x
		i64 lo = aEnd, hi = bEnd ;
		while ( lo < hi )
		{
			const i64 mid = ( lo + hi ) / 2 ;
			if ( t4_sortrec_less( recs[ src[mid] ], x, pool, idPool ) )
				lo = mid + 1 ;
			else
				hi = mid ;
		}
		dst[ i + ( lo - aEnd ) ] = src[i] ;
	}
	else
	{
		// right run: count the left run's elements that do not come after x
		i64 lo = base, hi = aEnd ;
		while ( lo < hi )
		{
			const i64 mid = ( lo + hi ) / 2 ;
			if ( !t4_sortrec_less( x, recs[ src[mid] ], pool, idPool ) )
				lo = mid + 1 ;
			else
				hi = mid ;
		}
		dst[ ( i - aEnd ) + lo ] = src[i] ;
	}
}

// ---- mate overlap detection (SURVEY.md 8f-3: "mate read-through / merge") -------------------------------------------------
// AlignAlgo::IsMateOverlap( fr, flen, sr, slen, minOverlap, offset, bestMatchCnt, checkTandem ) (AlignAlgo.hpp:1027-1096) as
// ProcessRead calls it for every read pair (main.cpp:264, 291): does a suffix of `fr` match a prefix of `sr` at exactly one
// offset (similarity threshold 0.85 ... 0.95 by length), and is the match not a tandem repeat?  One thread per pair.
// Verified on an H100 pair by pair against the reference: 300 000 pairs (more than one grid) and the function's edges.
struct T4MateParams
{
	u64 pool ;             // ASCII reads
	u64 fOff, sOff ;       // u64[n]
	u64 fLen, sLen ;       // i32[n]
	u64 minOverlap ;       // i32[n]
	u64 checkTandem ;      // u8[n]
	u64 overlapSize, offset, bestMatchCnt ; // i32[n] out; offset / bestMatchCnt as the function leaves them (-1 / -1 untouched)
	i64 n ;
} ;

T4_HD inline void t4_mate_overlap_one( const T4MateParams &P, i64 r )
{
	const char *fr = t4_x<char>( P.pool ) + t4_x<u64>( P.fOff )[r] ;
	const char *sr = t4_x<char>( P.pool ) + t4_x<u64>( P.sOff )[r] ;
	const int flen = t4_x<int32_t>( P.fLen )[r], slen = t4_x<int32_t>( P.sLen )[r] ;
	const int minOverlap = t4_x<int32_t>( P.minOverlap )[r] ;
	const bool checkTandem = t4_x<unsigned char>( P.checkTandem )[r] != 0 ;
	int i, j, k = 0 ;
	int bestMatchCnt = -1, offset = -1 ;
	int offsetCnt = 0 ;
	int overlapSize = -1 ;
	for ( j = 0 ; j < flen - minOverlap ; ++j )
	{
		int matchCnt = 0 ;
		bool flag = true ;
		double similarityThreshold = 0.95 ;
		if ( flen - j >= 100 )
			similarityThreshold = 0.85 ;
		else if ( flen - j >= 50 )
			similarityThreshold = 0.85 + ( flen - j - 50 ) / 50.0 * 0.1 ;
		for ( k = 0 ; j + k < flen && k < slen ; ++k )
		{
			if ( fr[j + k] == sr[k] )
				++matchCnt ;
			if ( matchCnt + ( flen - ( j + k ) - 1 ) < int( ( flen - j ) * similarityThreshold ) )
			{
				flag = false ;
				break ;
			}
		}
		if ( flag )
		{
			offset = j ;
			++offsetCnt ;
			overlapSize = k ;
			bestMatchCnt = matchCnt ;
		}
	}
	int ret = overlapSize ;
	if ( offsetCnt != 1 )
		ret = -1 ;
	else if ( checkTandem && overlapSize <= minOverlap * 2 )
	{
		for ( i = 1 ; i <= overlapSize / 2 && ret >= 0 ; ++i )
		{
			bool tandem = true ;
			for ( j = i ; j + i - 1 < overlapSize ; j += i )
			{
				for ( k = j ; k <= j + i - 1 ; ++k )
					if ( sr[k - j] != sr[k] )
						break ;
				if ( k <= j + i - 1 )
				{
					tandem = false ;
					break ;
				}
			}
			if ( tandem )
				ret = -1 ;
		}
	}
	t4_x<int32_t>( P.overlapSize )[r] = ret ;
	t4_x<int32_t>( P.offset )[r] = offset ;
	t4_x<int32_t>( P.bestMatchCnt )[r] = bestMatchCnt ;
}

#endif
