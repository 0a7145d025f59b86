// SeqSet::GetOverlapsFromRead on a REFERENCE gene set (SURVEY.md 8f-1, first half of the rough annotation:
// `refSet.AnnotateRead( read, 0, ... )` calls it per read, SeqSet.hpp:6050).  The assembly path only ever scores overlaps
// with novel contigs; reference sequences take the other branches of the same functions:
//
//   GetHitsFromRead            skipLimit = 0                                                   SeqSet.hpp:1351-1353
//   GetOverlapsFromHits        diagonal windows of `radius`, LongestIncreasingSubsequence      SeqSet.hpp:763-1063
//   GetVJOverlapsFromHits      the V-end / J-start rescue when no chain is long enough         SeqSet.hpp:1066-1160
//   GetOverlapsFromRead        strand of the best overlap, gaps between chain hits scored by the character-based affine
//                              AlignAlgo::GlobalAlignment, indels allowed, similarity >= refSeqSimilarity
//                                                                                              SeqSet.hpp:1508-2124, AlignAlgo.hpp:218-420
//
// STATUS: verified on an H100 against the compiled reference through t4_refset_get_overlaps and t4_refset_annotate
// (tests/test_gpu_preprocess.py: 528 workers on one read cursor, batch sizes around the worker count, the shipped example
// on the reference's hg38 gene set, interleaved scan / annotate / get-overlaps calls), and through the test emulation.  It
// runs in a kernel of its own (t4_annot_kernel).  Probe and key sort are the engine's collectives (c_ref_sorted_hits);
// everything after is serial per read on thread 0 in plain C (shared with the emulation).  The chain walk of a bucket is
// the stage-0 scan's t4_ref_bucket_chains (t4_refscan.h); overlaps are the engine's T4Ovl with its order, low-complexity
// and gene-name rules.
#ifndef T4_ANNOT_H
#define T4_ANNOT_H

#include "t4_refscan.h"

#define SCORE_GAPOPEN (-4)
#define SCORE_GAPEXTEND (-1)

struct T4AnnotScratch      // serial work space of one read (global memory), carved from one block by t4_annot_carve
{
	T4ScanScratch S ;      // bucket / window / LIS arrays (t4_refscan.h)
	int *hcA, *hcB ;       // chain pool: hitCoords of all overlaps
	int hcCap, hcUsed ;
	T4Ovl *ovl, *ovlTmp, *acc ; // acc: the overlaps of all contigs of a read (AnnotateRead)
	int ovlCap ;
	int *seqUsed ;         // int[nSeqs]
	int *ca, *cb ;         // contig intervals of the read (64 each)
	u64 *vj ;              // keys of the V-end / J-start hits (GetVJOverlapsFromHits)
	int *dpM, *dpE, *dpF ; // AlignAlgo::GlobalAlignment matrices
	signed char *align ;
	int dpCells, alignCap ;
	int overflow ;
} ;

T4_HD inline size_t t4_annot_scratch_bytes( int H, int gapLimit, int readLen, int nSeqs = 0 )
{
	const size_t h = (size_t)( H > 16 ? H : 16 ) ;
	const size_t g = (size_t)( gapLimit + 2 ) ;
	return 1024 + 8 * ( 2 * h ) + 4 * ( 6 * h ) + 4 * ( 2 * h ) + 3 * sizeof( T4Ovl ) * h + 8 * h + 3 * 4 * g * g + ( 2 * g + 2 * (size_t)readLen + 64 )
		+ 4 * (size_t)( nSeqs + 4 ) + 4 * 128 ;
}

T4_HD inline void t4_annot_carve( T4AnnotScratch &X, char *base, int H, int gapLimit, int readLen, int nSeqs = 0 )
{
	const size_t h = (size_t)( H > 16 ? H : 16 ) ;
	const size_t g = (size_t)( gapLimit + 2 ) ;
	char *p = base ;
	X.S.w = (u64 *)p ; p += 8 * 2 * h ;
	int *ia = (int *)p ; p += 4 * 6 * h ;
	X.S.ha = ia ; X.S.hb = ia + h ; X.S.top = ia + 2 * h ; X.S.link = ia + 3 * h ; X.S.oa = ia + 4 * h ; X.S.ob = ia + 5 * h ;
	X.hcA = (int *)p ; p += 4 * h ;
	X.hcB = (int *)p ; p += 4 * h ;
	X.hcCap = (int)h ; X.hcUsed = 0 ;
	p = (char *)( ( (uintptr_t)p + 15 ) & ~(uintptr_t)15 ) ;
	X.ovl = (T4Ovl *)p ; p += sizeof( T4Ovl ) * h ;
	X.ovlTmp = (T4Ovl *)p ; p += sizeof( T4Ovl ) * h ;
	X.acc = (T4Ovl *)p ; p += sizeof( T4Ovl ) * h ;
	X.ovlCap = (int)h ;
	X.seqUsed = (int *)p ; p += 4 * (size_t)( nSeqs + 4 ) ;
	X.ca = (int *)p ; p += 4 * 64 ;
	X.cb = (int *)p ; p += 4 * 64 ;
	p = (char *)( ( (uintptr_t)p + 15 ) & ~(uintptr_t)15 ) ;
	X.vj = (u64 *)p ; p += 8 * h ;
	X.dpM = (int *)p ; p += 4 * g * g ;
	X.dpE = (int *)p ; p += 4 * g * g ;
	X.dpF = (int *)p ; p += 4 * g * g ;
	X.dpCells = (int)( g * g ) ;
	X.align = (signed char *)p ;
	X.alignCap = (int)( 2 * g + 2 * (size_t)readLen + 32 ) ;
	X.overflow = 0 ;
}

// what the serial code needs to know about the gene set
struct T4RefView
{
	const T4Contig *seqs ;
	const char *A ;        // arena base
	int nSeqs ;
	int k, radius, hitLenRequired, nomatchGapLimit ;
	double refSeqSimilarity ;
	T4_HD const char *cons( int idx ) const { return A + seqs[idx].consOff + seqs[idx].lead ; }
	T4_HD const char *name( int idx ) const { return A + seqs[idx].nameOff ; }
	T4_HD int nameLen( int idx ) const { return seqs[idx].nameLen ; }
	T4_HD int len( int idx ) const { return seqs[idx].len ; }
} ;

// the view of the gene set cx is attached to
T4_D inline T4RefView t4_ref_view( T4Ctx &cx )
{
	const T4Stream *st = cx.st ;
	T4RefView V ;
	V.seqs = cx.P<T4Contig>( st->seqsOff ) ;
	V.A = cx.A ;
	V.nSeqs = st->nSeqs ;
	V.k = st->kmerLength ;
	V.radius = st->radius ;
	V.hitLenRequired = st->hitLenRequired ;
	V.nomatchGapLimit = st->nomatchGapLimit ;
	V.refSeqSimilarity = 0.75 ; // SeqSet.hpp:2566
	return V ;
}

// SeqSet::GetOverlapsFromHits for hits on reference sequences (SeqSet.hpp:763-1063): keys sorted by (strand, gene, a, b),
// each (strand, gene) bucket chained by t4_ref_bucket_chains.  filter / conservativeChain have no effect on a pure reference
// set (the filter statistics count novel sequences only and every posting list is below the `repeats` limit;
// conservativeChain is false for readType 0).  Appends to X.ovl from `first`; returns the new count.
T4_HD inline int t4_ref_overlaps_from_hits( const u64 *keys, int H, const T4RefView &V, int hitLenRequired, T4AnnotScratch &X, int first )
{
	int n = first ;
	for ( int i = 0 ; i < H ; )
	{
		const u64 g = keys[i] >> T4_KEY_IDX_SHIFT ;
		int j = i + 1 ;
		while ( j < H && ( keys[j] >> T4_KEY_IDX_SHIFT ) == g )
			++j ;
		const bool walked = t4_ref_bucket_chains( keys + i, j - i, V.k, V.radius, hitLenRequired, X.S, [&]( int lisSize, int hitLen ) {
			if ( n >= X.ovlCap || X.hcUsed + lisSize > X.hcCap )
			{
				X.overflow = 1 ;
				return false ;
			}
			T4Ovl &no = X.ovl[n] ;
			no.seqIdx = t4_key_idx( keys[i] ) ;
			no.readStart = X.S.oa[0] ;
			no.readEnd = X.S.oa[lisSize - 1] + V.k - 1 ;
			no.strand = t4_key_strand( keys[i] ) ;
			no.seqStart = X.S.ob[0] ;
			no.seqEnd = X.S.ob[lisSize - 1] + V.k - 1 ;
			no.matchCnt = 2 * hitLen ;
			no.indelCnt = 0 ;
			no.similarity = 0 ;
			no.hcStart = X.hcUsed ;
			no.hcCnt = lisSize ;
			no.infoFromHits = 0 ;
			for ( int x = 0 ; x < lisSize ; ++x )
			{
				X.hcA[X.hcUsed + x] = X.S.oa[x] ;
				X.hcB[X.hcUsed + x] = X.S.ob[x] ;
			}
			X.hcUsed += lisSize ;
			++n ;
			return true ;
		} ) ;
		if ( !walked ) // X.overflow
			return n ;
		i = j ;
	}
	return n ;
}

// SeqSet::GetVJOverlapsFromHits (SeqSet.hpp:1066-1160): chains of >= 17 bases among the hits on the last 31 bases of V genes
// and the first 31 of J genes; the best V + J pair of one chain type, V left of J on the read, survives.
T4_HD inline int t4_ref_vj_overlaps( const u64 *keys, int H, const T4RefView &V, T4AnnotScratch &X )
{
	int nv = 0 ;
	for ( int i = 0 ; i < H ; ++i )
	{
		const int idx = t4_key_idx( keys[i] ) ;
		const char c3 = V.name( idx )[3] ;
		const int b = t4_key_b( keys[i] ) ;
		if ( ( c3 == 'V' && b >= V.len( idx ) - 31 ) || ( c3 == 'J' && b < 31 ) )
			X.vj[nv++] = keys[i] ; // a subsequence of a sorted array: still sorted
	}
	X.hcUsed = 0 ;
	const int cnt = t4_ref_overlaps_from_hits( X.vj, nv, V, 17, X, 0 ) ;
	int maxMatchCnt = 0, tagi = 0, tagj = 0 ;
	for ( int i = 0 ; i < cnt ; ++i )
		for ( int j = i + 1 ; j < cnt ; ++j )
		{
			const char *ni = V.name( X.ovl[i].seqIdx ), *nj = V.name( X.ovl[j].seqIdx ) ;
			if ( ni[0] != nj[0] || ni[1] != nj[1] || ni[2] != nj[2] || ni[3] == nj[3] )
				continue ;
			if ( ni[3] == 'V' )
			{
				if ( X.ovl[i].readStart > X.ovl[j].readStart )
					continue ;
			}
			else if ( X.ovl[i].readStart < X.ovl[j].readStart )
				continue ;
			if ( X.ovl[i].matchCnt + X.ovl[j].matchCnt > maxMatchCnt )
			{
				maxMatchCnt = X.ovl[i].matchCnt + X.ovl[j].matchCnt ;
				tagi = i ;
				tagj = j ;
			}
		}
	if ( maxMatchCnt == 0 )
		return 0 ;
	const T4Ovl a = X.ovl[tagi], b = X.ovl[tagj] ;
	X.ovl[0] = a ;
	X.ovl[1] = b ;
	return 2 ;
}

// AlignAlgo::GlobalAlignment (AlignAlgo.hpp:218-420): banded affine-gap global alignment of characters; N matches anything.
// Only the edit counts are consumed (GetAlignStats), but they depend on the traceback, so all of it is restated.
T4_HD inline bool t4_ga_eq( char t, char p ) { return t == p || t == 'N' || p == 'N' ; }

T4_HD inline int t4_global_alignment( const char *t, int lent, const char *p, int lenp, T4AnnotScratch &X, int count[3] )
{
	count[0] = count[1] = count[2] = 0 ;
	if ( lent == 0 || lenp == 0 )
		return 0 ;
	if ( lent == 1 && lenp == 1 )
	{
		if ( t4_ga_eq( t[0], p[0] ) )
		{
			count[0] = 1 ;
			return SCORE_MATCH ;
		}
		count[1] = 1 ;
		return SCORE_MISMATCH ;
	}
	if ( ( lent + 1 ) * ( lenp + 1 ) > X.dpCells || lent + lenp + 2 > X.alignCap )
	{
		X.overflow = 1 ;
		return 0 ;
	}
	int *m = X.dpM, *e = X.dpE, *f = X.dpF ;
	int leftBand = 5, rightBand = 5 ;
	if ( lent > lenp )
		rightBand += lent - lenp ;
	else if ( lent < lenp )
		leftBand += lenp - lent ;
	int i, j ;
	const int negInf = ( lent + 1 ) * ( lenp + 1 ) * SCORE_GAPOPEN ;
	const int bmax = lent + 1 ;
	m[0] = e[0] = f[0] = 0 ;
	for ( i = 1 ; i <= lenp ; ++i )
	{
		e[i * bmax + 0] = SCORE_GAPOPEN + i * SCORE_GAPEXTEND ;
		f[i * bmax + 0] = SCORE_GAPOPEN + i * SCORE_GAPOPEN ;
		m[i * bmax + 0] = SCORE_GAPOPEN + i * SCORE_GAPOPEN ;
	}
	for ( j = 1 ; j <= lent ; ++j )
	{
		f[0 + j] = SCORE_GAPOPEN + j * SCORE_GAPEXTEND ;
		e[0 + j] = SCORE_GAPOPEN + i * SCORE_GAPOPEN ; // `i` (= lenp + 1 here), as in the reference (AlignAlgo.hpp:268)
		m[0 + j] = SCORE_GAPOPEN + j * SCORE_GAPOPEN ;
	}
	for ( i = 1 ; i <= lenp ; ++i )
	{
		const int start = ( i - leftBand < 1 ) ? 1 : ( i - leftBand ) ;
		const int end = ( i + rightBand > lent ) ? lent : ( i + rightBand ) ;
		if ( start > 1 )
		{
			j = start - 1 ;
			e[i * bmax + j] = f[i * bmax + j] = m[i * bmax + j] = negInf ;
		}
		if ( end < lent )
		{
			j = end + 1 ;
			e[i * bmax + j] = f[i * bmax + j] = m[i * bmax + j] = negInf ;
		}
		for ( j = start ; j <= end ; ++j )
		{
			int score = e[( i - 1 ) * bmax + j] + SCORE_GAPEXTEND ;
			int alt = m[( i - 1 ) * bmax + j] + SCORE_GAPOPEN + SCORE_GAPEXTEND ;
			if ( alt > score ) score = alt ;
			e[i * bmax + j] = score ;
			score = f[i * bmax + j - 1] + SCORE_GAPEXTEND ;
			alt = m[i * bmax + j - 1] + SCORE_GAPOPEN + SCORE_GAPEXTEND ;
			if ( alt > score ) score = alt ;
			f[i * bmax + j] = score ;
			score = m[( i - 1 ) * bmax + j - 1] + ( t4_ga_eq( t[j - 1], p[i - 1] ) ? SCORE_MATCH : SCORE_MISMATCH ) ;
			if ( e[i * bmax + j] > score ) score = e[i * bmax + j] ;
			if ( f[i * bmax + j] > score ) score = f[i * bmax + j] ;
			m[i * bmax + j] = score ;
		}
	}
	const int ret = m[lenp * bmax + lent] ;
	int tagi = lenp, tagj = lent, mat = 0 ;
	while ( tagi > 0 || tagj > 0 )
	{
		if ( mat == 0 )
		{
			const int mx = e[tagi * bmax + tagj] ;
			int a = EDIT_INSERT ;
			if ( f[tagi * bmax + tagj] >= mx )
				a = EDIT_DELETE ;
			if ( tagi > 0 && tagj > 0
				&& ( m[( tagi - 1 ) * bmax + tagj - 1] + ( t4_ga_eq( t[tagj - 1], p[tagi - 1] ) ? SCORE_MATCH : SCORE_MISMATCH ) == m[tagi * bmax + tagj] ) )
				a = t4_ga_eq( t[tagj - 1], p[tagi - 1] ) ? EDIT_MATCH : EDIT_MISMATCH ;
			if ( a == EDIT_MATCH || a == EDIT_MISMATCH )
			{
				++count[a == EDIT_MATCH ? 0 : 1] ;
				--tagi ; --tagj ;
			}
			else if ( a == EDIT_INSERT )
				mat = 1 ;
			else
				mat = 2 ;
		}
		else if ( mat == 1 )
		{
			++count[2] ;
			if ( tagi > 0 )
			{
				if ( m[( tagi - 1 ) * bmax + tagj] + SCORE_GAPOPEN + SCORE_GAPEXTEND == e[tagi * bmax + tagj] )
					mat = 0 ;
				--tagi ;
			}
			else
				mat = 2 ;
		}
		else
		{
			++count[2] ;
			if ( tagj > 0 )
			{
				if ( m[tagi * bmax + tagj - 1] + SCORE_GAPOPEN + SCORE_GAPEXTEND == f[tagi * bmax + tagj] )
					mat = 0 ;
				--tagj ;
			}
			else
				mat = 1 ;
		}
	}
	return ret ;
}

// std::sort( overlaps ), serial
T4_HD inline void t4_ovl_sort( T4Ovl *o, T4Ovl *tmp, int n )
{
	for ( int i = 0 ; i < n ; ++i )
		tmp[t4_ovl_rank( o, n, i )] = o[i] ;
	for ( int i = 0 ; i < n ; ++i )
		o[i] = tmp[i] ;
}

// SeqSet::GetOverlapsFromRead( read, 0, -1, readType 0, false ) on a reference set, from the sorted hits on: chains (or the
// V/J rescue), overlap order, strand of the best, scoring, similarity filter.  read / rc: the read and its reverse
// complement.  The overlaps end in X.ovl[0..ret); returns their number (0: none).
T4_HD inline int t4_ref_overlaps_from_read( const u64 *keys, int H, const char *read, const char *rc, int len, const T4RefView &V, T4AnnotScratch &X )
{
	X.hcUsed = 0 ;
	int overlapCnt = t4_ref_overlaps_from_hits( keys, H, V, V.hitLenRequired, X, 0 ) ;
	if ( X.overflow )
		return 0 ;
	if ( overlapCnt == 0 )
	{
		overlapCnt = t4_ref_vj_overlaps( keys, H, V, X ) ;
		if ( overlapCnt == 0 || X.overflow )
			return 0 ;
	}
	t4_ovl_sort( X.ovl, X.ovlTmp, overlapCnt ) ;
	{
		int kk = 1 ;
		for ( int i = 1 ; i < overlapCnt ; ++i ) // readType 0: keep the strand of the best overlap (SeqSet.hpp:1601-1616)
		{
			if ( X.ovl[i].strand != X.ovl[0].strand )
				continue ;
			if ( i != kk )
				X.ovl[kk] = X.ovl[i] ;
			++kk ;
		}
		overlapCnt = kk ;
	}
	const int k = V.k ;
	for ( int i = 0 ; i < overlapCnt ; ++i )
	{
		T4Ovl &o = X.ovl[i] ;
		const char *r = o.strand == 1 ? read : rc ;
		const char *cons = V.cons( o.seqIdx ) ;
		o.infoFromHits = i ;
		const int *ha = X.hcA + o.hcStart, *hb = X.hcB + o.hcStart ;
		int matchCnt = 2 * k, mismatchCnt = 0, indelCnt = 0 ;
		double similarity = 1 ;
		for ( int j = 1 ; j < o.hcCnt ; ++j )
		{
			if ( hb[j - 1] - ha[j - 1] == hb[j] - ha[j] )
			{
				if ( ha[j - 1] + k - 1 >= ha[j] )
					matchCnt += 2 * ( ha[j] - ha[j - 1] ) ;
				else
				{
					matchCnt += 2 * k ;
					if ( hb[j] - ( hb[j - 1] + k ) > V.nomatchGapLimit || ha[j] - ( ha[j - 1] + k ) > V.nomatchGapLimit )
					{
						similarity = 0 ;
						break ;
					}
					int count[3] ;
					t4_global_alignment( cons + hb[j - 1] + k, hb[j] - ( hb[j - 1] + k ), r + ha[j - 1] + k, ha[j] - ( ha[j - 1] + k ), X, count ) ;
					matchCnt += 2 * count[0] ;
					mismatchCnt += count[1] ;
					indelCnt += count[2] ;
					if ( V.radius == 0 && indelCnt > 0 )
					{
						similarity = 0 ;
						break ;
					}
				}
			}
			else
			{
				if ( V.radius == 0 )
				{
					similarity = 0 ;
					break ;
				}
				if ( ha[j - 1] + k - 1 >= ha[j] && hb[j - 1] + k - 1 < hb[j] )
				{
					matchCnt += 2 * ( ha[j] - ha[j - 1] ) ;
					indelCnt += ( hb[j] - ( hb[j - 1] + k ) + ( ha[j] + k - ha[j - 1] ) ) ;
				}
				else if ( ha[j - 1] + k - 1 < ha[j] && hb[j - 1] + k - 1 >= hb[j] )
				{
					matchCnt += 2 * ( hb[j] - hb[j - 1] ) ;
					indelCnt += ( ha[j] - ( ha[j - 1] + k ) + ( hb[j] + k - hb[j - 1] ) ) ;
				}
				else if ( ha[j - 1] + k - 1 >= ha[j] && hb[j - 1] + k - 1 >= hb[j] )
				{
					const int da = ha[j] - ha[j - 1], db = hb[j] - hb[j - 1] ;
					matchCnt += 2 * ( da < db ? da : db ) ;
					const int dd = ( ha[j] - hb[j] ) - ( ha[j - 1] - hb[j - 1] ) ;
					indelCnt += dd > 0 ? dd : -dd ;
				}
				else
				{
					matchCnt += 2 * k ;
					if ( hb[j] - ( hb[j - 1] + k ) > V.nomatchGapLimit || ha[j] - ( ha[j - 1] + k ) > V.nomatchGapLimit )
					{
						similarity = 0 ;
						break ;
					}
					int count[3] ;
					t4_global_alignment( cons + hb[j - 1] + k, hb[j] - ( hb[j - 1] + k ), r + ha[j - 1] + k, ha[j] - ( ha[j - 1] + k ), X, count ) ;
					matchCnt += 2 * count[0] ;
					mismatchCnt += count[1] ;
					indelCnt += count[2] ;
				}
			}
		}
		(void)mismatchCnt ;
		o.matchCnt = matchCnt ;
		o.indelCnt = indelCnt ;
		if ( similarity == 1 )
			o.similarity = (double)matchCnt / ( o.seqEnd - o.seqStart + 1 + o.readEnd - o.readStart + 1 ) ;
		else
			o.similarity = 0 ;
		if ( t4_low_complex( r, o ) )
			o.similarity = 0 ;
	}
	int kk = 0 ;
	for ( int i = 0 ; i < overlapCnt ; ++i )
	{
		if ( X.ovl[i].similarity < V.refSeqSimilarity )
			continue ;
		if ( kk != i )
			X.ovl[kk] = X.ovl[i] ;
		++kk ;
	}
	return kk ;
}

// ---- SeqSet::AnnotateRead( read, 0, geneOverlap, NULL, NULL ) (SeqSet.hpp:6016-6340, the detailLevel 0 statements) ----------
// SeqSet::GetContigIntervals (SeqSet.hpp:5289-5321): the read is cut where gapN = 7 N's fall into a window of 7
T4_HD inline int t4_contig_intervals( const char *read, int len, int *ca, int *cb, int cap )
{
	const int gapN = 7 ;
	int n = 0 ;
	for ( int i = 0 ; i < len ; )
	{
		int NCnt = 0, j ;
		for ( j = i + 1 ; j < len ; ++j )
		{
			if ( j >= i + gapN && read[j - gapN] == 'N' )
				--NCnt ;
			if ( read[j] == 'N' )
				++NCnt ;
			if ( NCnt >= gapN )
				break ;
		}
		if ( n >= cap )
			return -1 ;
		ca[n] = i ;
		cb[n] = j < len ? j - gapN : j - 1 ;
		++n ;
		if ( j >= len )
			break ;
		i = j + 1 ;
	}
	return n ;
}

// From the overlaps of all contigs (read coordinates already shifted, each contig's list sorted) to geneOverlap[4]
// (V, D, J, C): SeqSet.hpp:6230-6340 without the detailLevel >= 1 statements.  ovl is reordered in place.
T4_HD inline int t4_annotate_select( T4Ovl *ovl, T4Ovl *tmp, int overlapCnt, int *seqUsed, int len, const T4RefView &V, T4Ovl geneOverlap[4] )
{
	for ( int t = 0 ; t < 4 ; ++t )
	{
		geneOverlap[t].seqIdx = -1 ;
		geneOverlap[t].readStart = geneOverlap[t].readEnd = geneOverlap[t].seqStart = geneOverlap[t].seqEnd = -1 ; // _overlap()
		geneOverlap[t].strand = 1 ;
		geneOverlap[t].matchCnt = 0 ;
		geneOverlap[t].indelCnt = 0 ;
		geneOverlap[t].similarity = 0 ;
		geneOverlap[t].infoFromHits = 0 ;
		geneOverlap[t].hcStart = geneOverlap[t].hcCnt = 0 ;
		geneOverlap[t].preMatchCnt = 0 ;
	}
	t4_ovl_sort( ovl, tmp, overlapCnt ) ;
	for ( int i = 0 ; i < V.nSeqs ; ++i )
		seqUsed[i] = -1 ;
	const double geneSimilarity = 0.8 ;
	int k = 0 ;
	for ( int i = 0 ; i < overlapCnt ; ++i )
	{
		const int geneType = t4_gene_type( V.name( ovl[i].seqIdx ), V.nameLen( ovl[i].seqIdx ) ) ;
		if ( geneType < 0 || geneType == 1 )
			continue ;
		if ( seqUsed[ ovl[i].seqIdx ] == -1 && ovl[i].similarity >= geneSimilarity )
		{
			seqUsed[ ovl[i].seqIdx ] = k ;
			ovl[k] = ovl[i] ;
			++k ;
		}
		else if ( seqUsed[ ovl[i].seqIdx ] != -1 && geneType == 2 )
		{
			T4Ovl &baseline = ovl[ seqUsed[ ovl[i].seqIdx ] ] ;
			if ( ovl[i].matchCnt == baseline.matchCnt && ovl[i].similarity == baseline.similarity )
			{
				int j ;
				for ( j = 0 ; j < k ; ++j )
					if ( t4_gene_type( V.name( ovl[j].seqIdx ), V.nameLen( ovl[j].seqIdx ) ) == 3 )
						break ;
				if ( j < k && ovl[i].readEnd <= ovl[j].readStart + 3 )
				{
					const int d1 = ovl[i].readEnd - ovl[j].readStart, d2 = baseline.readEnd - ovl[j].readStart ;
					if ( baseline.readEnd > ovl[j].readStart + 3 || ( d1 < 0 ? -d1 : d1 ) < ( d2 < 0 ? -d2 : d2 ) )
						baseline = ovl[i] ;
				}
			}
		}
	}
	overlapCnt = k ;
	if ( overlapCnt == 0 )
		return 0 ;
	char BT = '\0', chain = '\0' ;
	for ( int i = 0 ; i < overlapCnt ; ++i )
	{
		const char *name = V.name( ovl[i].seqIdx ) ;
		if ( BT && name[0] != BT )
			continue ;
		BT = name[0] ;
		if ( chain && !( name[2] == chain || ( name[2] == 'D' && chain == 'A' ) || ( name[2] == 'A' && chain == 'D' ) ) )
			continue ;
		chain = name[2] ;
		const int geneType = t4_gene_type( name, V.nameLen( ovl[i].seqIdx ) ) ;
		if ( geneType >= 0 && geneOverlap[geneType].seqIdx == -1 )
			geneOverlap[geneType] = ovl[i] ;
	}
	// a short constant-gene match next to a V / J match that overlaps it is taken for random (SeqSet.hpp:6308-6323)
	if ( geneOverlap[3].seqIdx != -1 && geneOverlap[3].readEnd - geneOverlap[3].readStart + 1 <= len / 2
		&& geneOverlap[3].readEnd - geneOverlap[3].readStart + 1 <= 50 )
	{
		for ( int i = 0 ; i < 3 ; ++i )
			if ( geneOverlap[i].seqIdx >= 0
				&& ( geneOverlap[i].readEnd - 17 > geneOverlap[3].readStart || geneOverlap[3].readEnd < geneOverlap[i].readEnd )
				&& geneOverlap[3].seqStart >= 100 )
			{
				geneOverlap[3].seqIdx = -1 ;
				break ;
			}
	}
	return 1 ;
}

// ---- T4_OP_REF_OVERLAPS: one read against the gene set (the per-call entry; body of t4_annot_kernel) ------------------
struct T4RefOvlParams
{
	u64 scratch ;          // device block of scratchBytes
	u64 scratchBytes ;
	int hMax ;             // the scratch was sized for this many hits
	int pad ;
} ;

T4_D inline void c_ref_get_overlaps( T4Ctx &cx, T4Op *op )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	const T4RefOvlParams *P = t4_x<T4RefOvlParams>( op->out2 ) ;
	c_load_read( cx, t4_x<char>( op->read ), op->len ) ;
	int ret = -1 ;
	if ( op->len >= st->kmerLength )
	{
		ret = 0 ;
		const u64 *sorted = 0 ;
		bool failed ;
		const u32 H = c_ref_sorted_hits( cx, op->len, P->hMax, 7, &sorted, failed ) ;
		if ( H > 0 )
		{
			if ( cx.tid == 0 )
			{
				T4AnnotScratch X ;
				t4_annot_carve( X, t4_x<char>( P->scratch ), (int)H, st->nomatchGapLimit, op->len ) ;
				const T4RefView V = t4_ref_view( cx ) ;
				int n = t4_ref_overlaps_from_read( sorted, (int)H, sm->read, sm->rc, op->len, V, X ) ;
				if ( X.overflow )
					t4_raise( cx, T4_E_NOMEM, 8 ) ;
				int32_t *out = t4_x<int32_t>( op->out ) ;
				double *sim = (double *)( out + 8 * op->outCap ) ;
				for ( int i = 0 ; i < n && i < op->outCap ; ++i )
				{
					const T4Ovl &o = X.ovl[i] ;
					out[8 * i] = o.seqIdx ; out[8 * i + 1] = o.readStart ; out[8 * i + 2] = o.readEnd ; out[8 * i + 3] = o.seqStart ;
					out[8 * i + 4] = o.seqEnd ; out[8 * i + 5] = o.strand ; out[8 * i + 6] = o.matchCnt ; out[8 * i + 7] = o.indelCnt ;
					sim[i] = o.similarity ;
				}
				sm->bi[0] = n ;
			}
			T4_SYNC() ;
			ret = sm->bi[0] ;
			T4_SYNC() ;
		}
	}
	if ( cx.tid == 0 )
		op->ret = cx.st->error ? cx.st->error : ret ;
}

// ---- T4_OP_REF_ANNOTATE: worker loop, AnnotateRead( read, 0, ... ) for a batch of reads --------------------------------------
struct T4AnnotParams
{
	u64 pool, seqOff, len ;   // reads (device): ASCII pool, u64[n], i32[n]
	u64 out ;                 // int32[n][4][8]: per gene type V, D, J, C: seqIdx (-1: none), readStart, readEnd, seqStart, seqEnd, strand, matchCnt, indelCnt
	u64 sim ;                 // double[n][4]
	u64 cursor ;              // u64[4]
	u64 setOff ;              // the gene set's stream
	u64 scratch ;             // per worker blocks of scratchStride bytes
	u64 scratchStride ;
	i64 n ;
	int hMax ;
	int pad ;
} ;

T4_D inline void c_ref_annotate( T4Ctx &cx, T4Op *op )
{
	const T4AnnotParams *P = t4_x<T4AnnotParams>( op->out ) ;
	T4Smem *sm = cx.sm ;
	T4Stream *st = cx.st ;
	const u64 *seqOff = t4_x<u64>( P->seqOff ) ;
	const int32_t *lens = t4_x<int32_t>( P->len ) ;
	const char *pool = t4_x<char>( P->pool ) ;
	int32_t *out = t4_x<int32_t>( P->out ) ;
	double *sim = t4_x<double>( P->sim ) ;
	u64 *cursor = t4_x<u64>( P->cursor ) ;
	char *scratch = t4_x<char>( P->scratch ) + (u64)op->n * P->scratchStride ;
	c_assign_attach( cx, cx.P<T4Stream>( P->setOff ) ) ;
	const T4RefView V = t4_ref_view( cx ) ;
	bool failed = false ;
	while ( !failed )
	{
		T4_SYNC() ;
		if ( cx.tid == 0 )
			sm->bu[0] = t4_atomic_add( cursor, 1ull ) ;
		T4_SYNC() ;
		const i64 r = (i64)sm->bu[0] ;
		if ( r >= P->n )
			break ;
		const int len = lens[r] ;
		const char *src = pool + seqOff[r] ;
		if ( len > T4_DEV_MAX_READ )
		{
			if ( cx.tid == 0 )
				t4_raise( cx, T4_E_UNSUPPORTED, 5 ) ;
			failed = c_uniform_error( cx ) != 0 ;
			break ;
		}
		// contig intervals of the read (thread 0 reads it from global memory), broadcast through the scratch block
		T4AnnotScratch X ;
		t4_annot_carve( X, scratch, P->hMax, st->nomatchGapLimit, T4_DEV_MAX_READ, V.nSeqs ) ;
		if ( cx.tid == 0 )
			sm->bi[2] = t4_contig_intervals( src, len, X.ca, X.cb, 64 ) ;
		T4_SYNC() ;
		const int contigCnt = sm->bi[2] ;
		T4_SYNC() ;
		if ( contigCnt < 0 )
		{
			if ( cx.tid == 0 )
				t4_raise( cx, T4_E_UNSUPPORTED, 9 ) ;
			failed = c_uniform_error( cx ) != 0 ;
			break ;
		}
		int nAcc = 0 ; // thread 0
		for ( int c = 0 ; c < contigCnt && !failed ; ++c )
		{
			const int ca = X.ca[c], clen = X.cb[c] - X.ca[c] + 1 ;
			if ( clen < st->kmerLength )
				continue ; // GetOverlapsFromRead returns -1: no overlaps
			c_load_read( cx, src + ca, clen ) ;
			const u64 *sorted = 0 ;
			const u32 H = c_ref_sorted_hits( cx, clen, P->hMax, 7, &sorted, failed ) ;
			if ( failed )
				break ;
			if ( H > 0 && cx.tid == 0 )
			{
				const int n = t4_ref_overlaps_from_read( sorted, (int)H, sm->read, sm->rc, clen, V, X ) ;
				if ( X.overflow || nAcc + n > X.ovlCap )
					t4_raise( cx, T4_E_NOMEM, 8 ) ;
				else
				{
					// shift to read coordinates and sort this contig's list (SeqSet.hpp:6050-6057), then append
					for ( int i = 0 ; i < n ; ++i )
					{
						X.ovl[i].readStart += ca ;
						X.ovl[i].readEnd += ca ;
					}
					t4_ovl_sort( X.ovl, X.ovlTmp, n ) ;
					for ( int i = 0 ; i < n ; ++i )
						X.acc[nAcc + i] = X.ovl[i] ;
					nAcc += n ;
				}
			}
			failed = c_uniform_error( cx ) != 0 ;
		}
		if ( failed )
			break ;
		if ( cx.tid == 0 )
		{
			T4Ovl go[4] ;
			t4_annotate_select( X.acc, X.ovlTmp, nAcc, X.seqUsed, len, V, go ) ;
			for ( int t = 0 ; t < 4 ; ++t )
			{
				int32_t *o = out + ( r * 4 + t ) * 8 ;
				o[0] = go[t].seqIdx ; o[1] = go[t].readStart ; o[2] = go[t].readEnd ; o[3] = go[t].seqStart ; o[4] = go[t].seqEnd ;
				o[5] = go[t].strand ; o[6] = go[t].matchCnt ; o[7] = go[t].indelCnt ;
				sim[r * 4 + t] = go[t].similarity ;
			}
		}
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
		op->ret = cx.st->error ? cx.st->error : 0 ;
}

T4_D inline void c_run_annot_op( T4Ctx &cx, T4Op *op )
{
	T4Smem *sm = cx.sm ;
	if ( cx.tid == 0 )
		for ( int i = 0 ; i < T4_N_COUNTERS ; ++i )
			sm->ctr[i] = 0 ;
#if T4_CUDA
	if ( cx.tid == 0 )
	{
		for ( int i = 0 ; i < 8 ; ++i )
			sm->ph[i] = 0 ;
		sm->phCur = 0 ;
		sm->phLast = clock64() ;
	}
#endif
	T4_SYNC() ;
	if ( op->op == T4_OP_REF_OVERLAPS )
		c_ref_get_overlaps( cx, op ) ;
	else if ( op->op == T4_OP_REF_ANNOTATE )
		c_ref_annotate( cx, op ) ;
	T4_SYNC() ;
}

#endif
