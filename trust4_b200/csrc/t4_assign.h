// The AssignRead pass of the stage-1 driver on the device (SURVEY.md 8f-2):
//
//   SeqSet extendedSeq( k ) ; extendedSeq.InputSeqSet( seqSet, false ) ;          main.cpp:2047-2048, SeqSet.hpp:3108
//   extendedSeq.SetNovelSeqSimilarity( 0.95 ) ;                                    main.cpp:2074
//   for every assembled read: extendedSeq.AssignRead( read, strand, barcode, assign ) ;  main.cpp:2075-2116, SeqSet.hpp:4632
//   extendedSeq.SetNovelSeqSimilarity( 0.9 ) ; extendedSeq.RecomputePosWeight( assembledReads ) ;  main.cpp:2117-2118, SeqSet.hpp:4705
//
// AssignRead only READS the extended set, so -- unlike AddRead -- the pass is not a serial chain: it runs as three
// launches of the auxiliary kernel (t4_aux_kernel, same (tid, nt, barrier) engine as the stream kernel):
//   PREP      one CTA per set: build the extended set from the stage-1 set and lay out the list of assembled reads
//             (main pass in order, then the rescued ones) with, for every list slot, the slot whose result it shares
//             (identical neighbouring read strings reuse the previous result, main.cpp:2078-2081);
//   ASSIGN    worker CTAs over the WHOLE GPU: a worker owns only scratch (a T4Stream shell), takes list slots from an
//             atomic cursor, attaches to the slot's set and runs GetOverlapsFromRead + ExtendOverlap for that read;
//   RECOMPUTE one CTA per set: RecomputePosWeight from the assignments (integer atomics: order independent).
#ifndef T4_ASSIGN_H
#define T4_ASSIGN_H

#include "t4_engine.h"

struct T4AssignParams      // device resident; every CTA of the three launches reads it through T4Op::out
{
	u64 descs ;            // t4_read_desc[nDescs]   (absolute pointers, like T4Op)
	u64 pool ;             // ASCII read pool
	u64 ret, strands, rescue ; // results of the assembly run: int32[nDescs], int8[nDescs], int32[nDescs]
	u64 list ;             // int32[nDescs]: set j owns slots [descOff[j], descOff[j+1]); the first listCnt[j] hold record indices
	u64 leader ;           // int32[nDescs]: slot whose AssignRead result this slot takes (itself: AssignRead is called)
	u64 slotSet ;          // u32[nDescs]
	u64 assign ;           // int32[8 * nDescs] by RECORD: seqIdx, readStart, readEnd, seqStart, seqEnd, strand, matchCnt, 0
	u64 sim ;              // double[nDescs] by record
	u64 extOff ;           // u64[nSets]: arena offsets of the extended sets
	u64 srcOff ;           // u64[nSets]: arena offsets of the stage-1 sets
	u64 descOff ;          // i64[nSets + 1]
	u64 listCnt ;          // u32[nSets]
	u64 cursor ;           // u64[4]: [0] slot cursor of the ASSIGN launch, [1] AssignRead calls, [2] reads assigned, [3] list length
	i64 nDescs ;
	int nSets ;
	int kmerLength ;
} ;

#define T4_ASSIGN_CHUNK 8          /* list slots per cursor step */

// st->error as ONE value for the whole CTA: a thread may raise an error after the last barrier of a collective, so
// control flow that leads to barriers must not branch on each thread's own load of it.
T4_D inline int c_uniform_error( T4Ctx &cx )
{
	T4_SYNC() ;
	if ( cx.tid == 0 )
		cx.sm->bi[1] = cx.st->error ;
	T4_SYNC() ;
	const int e = cx.sm->bi[1] ;
	T4_SYNC() ;
	return e ;
}

// ---- PREP --------------------------------------------------------------------------------------------------------
// SeqSet::InputSeqSet( in, false ), SeqSet.hpp:3108-3139: every live contig of `src`, in slot order, becomes the next
// slot of this (fresh) set -- consensus, posWeight, anchors, numRead, barcode, name -- and is indexed at this set's k
// unless it was purged (seqs[i].index == false).
T4_D inline void c_input_seqset( T4Ctx &cx, const T4Stream *src )
{
	T4Smem *sm = cx.sm ;
	const int n = src->nSeqs ;
	for ( int s = 0 ; s < n ; ++s )
	{
		const T4Contig *sc = cx.P<T4Contig>( src->seqsOff ) + s ;
		if ( sc->consOff == 0 )
			continue ;
		T4_SYNC() ;
		if ( cx.tid == 0 )
		{
			s_refill_slab( cx ) ;
			int idx = s_new_contig( cx, sc->len ) ;
			if ( idx >= 0 )
			{
				T4Contig *c = t4_seq( cx, idx ) ;
				s_set_name( cx, c, cx.P<char>( sc->nameOff ), sc->nameLen ) ;
				c->barcode = sc->barcode ;
				c->numRead = sc->numRead ;
				c->minLeftExtAnchor = sc->minLeftExtAnchor ;
				c->minRightExtAnchor = sc->minRightExtAnchor ;
				c->flags = sc->flags ;
			}
			sm->bi[0] = idx ;
		}
		T4_SYNC() ;
		const int idx = sm->bi[0] ;
		T4_SYNC() ;
		if ( idx < 0 || c_uniform_error( cx ) )
			return ;
		T4Contig *c = t4_seq( cx, idx ) ;
		char *cons = t4_cons( cx, c ) ;
		int *pw = t4_pw( cx, c ) ;
		const char *scons = cx.P<char>( sc->consOff ) + sc->lead ;
		const int *spw = cx.P<int>( sc->pwOff ) + 4 * sc->lead ;
		unsigned char *eq = t4_eq( cx, c ) ;
		const unsigned char *seqb = cx.P<unsigned char>( sc->pwOff + 16ull * sc->cap ) + sc->lead ;
		const int len = sc->len ;
		T4_PAR_FOR( i, len )
		{
			cons[i] = scons[i] ;
			eq[i] = seqb[i] ;
		}
		T4_PAR_FOR( i, 4 * len )
			pw[i] = spw[i] ;
		T4_SYNC() ;
		if ( !( sc->flags & T4_CF_NOINDEX ) )
			c_index_op( cx, cons, len, T4_IDX_BUILD, idx, sc->barcode, 0, 0 ) ;
	}
	T4_SYNC() ;
}

T4_D inline bool t4_same_read( const t4_read_desc &a, const t4_read_desc &b, const char *pool )
{
	if ( a.len != b.len )
		return false ;
	if ( a.seq_off == b.seq_off )
		return true ;
	const char *x = pool + a.seq_off, *y = pool + b.seq_off ;
	for ( int i = 0 ; i < a.len ; ++i )
		if ( x[i] != y[i] )
			return false ;
	return true ;
}

// Stable compaction of the records of [lo, hi) that satisfy `rescued ? rescue[i] >= 0 : ret[i] >= 0` into list[base...].
// Collective; returns the number appended.
T4_D inline int c_assign_compact( T4Ctx &cx, const T4AssignParams *P, i64 lo, i64 hi, bool rescued, i64 base )
{
	const int32_t *ret = t4_x<int32_t>( P->ret ), *resc = t4_x<int32_t>( P->rescue ) ;
	int32_t *list = t4_x<int32_t>( P->list ) ;
	const i64 n = hi - lo ;
	const i64 chunk = ( n + cx.nt - 1 ) / cx.nt ;
	i64 a = lo + chunk * cx.tid, b = a + chunk ;
	if ( a > hi ) a = hi ;
	if ( b > hi ) b = hi ;
	u32 c = 0 ;
	for ( i64 i = a ; i < b ; ++i )
		if ( rescued ? ( resc[i] != INT32_MIN && resc[i] >= 0 ) : ( ret[i] >= 0 ) )
			++c ;
	u32 total ;
	u32 o = c_scan_threads( cx, c, total ) ;
	for ( i64 i = a ; i < b ; ++i )
		if ( rescued ? ( resc[i] != INT32_MIN && resc[i] >= 0 ) : ( ret[i] >= 0 ) )
			list[base + o++] = (int32_t)i ;
	T4_SYNC() ;
	return (int)total ;
}

T4_D inline void c_assign_prep( T4Ctx &cx, T4Op *op )
{
	const T4AssignParams *P = t4_x<T4AssignParams>( op->out ) ;
	T4Smem *sm = cx.sm ;
	const int j = op->n ;
	const T4Stream *src = cx.P<T4Stream>( t4_x<u64>( P->srcOff )[j] ) ;
	c_input_seqset( cx, src ) ;
	if ( cx.tid == 0 )
		cx.st->novelSeqSimilarity = 0.95 ; // main.cpp:2074
	const i64 lo = t4_x<i64>( P->descOff )[j], hi = t4_x<i64>( P->descOff )[j + 1] ;
	// the assembled reads in the driver's order: main pass (main.cpp:1779), then the rescue pass (main.cpp:1933)
	int cnt = c_assign_compact( cx, P, lo, hi, false, lo ) ;
	if ( P->rescue )
		cnt += c_assign_compact( cx, P, lo, hi, true, lo + cnt ) ;
	int32_t *list = t4_x<int32_t>( P->list ), *leader = t4_x<int32_t>( P->leader ) ;
	u32 *slotSet = t4_x<u32>( P->slotSet ) ;
	int32_t *assign = t4_x<int32_t>( P->assign ) ;
	double *sim = t4_x<double>( P->sim ) ;
	for ( i64 i = lo + cx.tid ; i < hi ; i += cx.nt )
	{
		if ( i >= lo + cnt )
		{
			list[i] = -1 ;
			leader[i] = -1 ;
		}
		slotSet[i] = (u32)j ;
		for ( int x = 0 ; x < 8 ; ++x )
			assign[8 * i + x] = x == 0 ? T4_ASSIGN_NOT_LISTED : 0 ;
		sim[i] = 0.0 ;
	}
	T4_SYNC() ;
	// leader of a slot: the closest slot at or before it whose read string differs from its predecessor's
	// (main.cpp:2078: `i == 0 || strcmp( read[i], read[i - 1] )`)
	const t4_read_desc *descs = t4_x<t4_read_desc>( P->descs ) ;
	const char *pool = t4_x<char>( P->pool ) ;
	const int chunk = ( cnt + cx.nt - 1 ) / cx.nt ;
	int a = chunk * cx.tid, b = a + chunk ;
	if ( a > cnt ) a = cnt ;
	if ( b > cnt ) b = cnt ;
	int last = -1 ;
	for ( int p = a ; p < b ; ++p )
	{
		const bool head = p == 0 || !t4_same_read( descs[ list[lo + p] ], descs[ list[lo + p - 1] ], pool ) ;
		if ( head )
			last = p ;
		leader[lo + p] = head ? (int32_t)( lo + p ) : -1 ;
	}
	sm->scan[cx.tid] = (u32)last ;
	T4_SYNC() ;
	int carry = -1 ;
	for ( int t = 0 ; t < cx.tid ; ++t )
		if ( (int)sm->scan[t] > carry )
			carry = (int)sm->scan[t] ;
	T4_SYNC() ;
	u32 heads = 0 ;
	for ( int p = a ; p < b ; ++p )
	{
		if ( leader[lo + p] >= 0 )
		{
			carry = p ;
			++heads ;
		}
		else
			leader[lo + p] = (int32_t)( lo + carry ) ;
	}
	u32 totalHeads ;
	c_scan_threads( cx, heads, totalHeads ) ;
	if ( cx.tid == 0 )
	{
		t4_x<u32>( P->listCnt )[j] = (u32)cnt ;
		t4_atomic_add( t4_x<u64>( P->cursor ) + 1, (u64)totalHeads ) ;
		t4_atomic_add( t4_x<u64>( P->cursor ) + 3, (u64)cnt ) ;
		op->ret = cnt ;
	}
	T4_SYNC() ;
}

// ---- ASSIGN ------------------------------------------------------------------------------------------------------
// int SeqSet::AssignRead( read, strand, barcode, assign ), SeqSet.hpp:4632-4702, novel-contig set.  Collective; the read
// is in cx.sm->read / rc.  Returns the contig slot (result in cx.sm->e0) or -1.
T4_D inline int c_assign_read( T4Ctx &cx, int len, int strand, int barcode )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	int overlapCnt = c_get_overlaps( cx, len, strand, barcode, false ) ;
	T4_PHASE( cx, 0 ) ;
	if ( c_uniform_error( cx ) || overlapCnt <= 0 || st->nSeqs == 0 )
		return -1 ;
	c_sort_overlaps( cx, overlapCnt ) ; // std::sort( overlaps ), SeqSet.hpp:4649
	T4Ovl *overlaps = cx.P<T4Ovl>( st->ovlOff ) ;
	const char *r = ( overlaps[0].strand == 1 ) ? sm->read : sm->rc ;
	const double factor = barcode == -1 ? 1.0 : 2.0 ; // SeqSet.hpp:4678
	// ExtendOverlap is a pure function of (overlap, read, contig): all overlaps at once, then the first in order that
	// extends over the whole read wins (SeqSet.hpp:4674-4690)
	u32 *bits = cx.P<u32>( st->bitsOff ) ;
	c_overhang_bits( cx, overlaps, overlapCnt, r, len, bits ) ;
	T4SideStats *sstats = (T4SideStats *)cx.P<char>( st->failOff ) ;
	T4DpScratch ds = t4_dp_scratch( cx ) ;
	T4_PAR_FOR( x, 2 * overlapCnt )
	{
		const int i = x >> 1, right = x & 1 ;
		const T4Ovl &o = overlaps[i] ;
		T4Contig *seq = t4_seq( cx, o.seqIdx ) ;
		int *pw = t4_pw( cx, seq ) ;
		T4AlignView av ;
		if ( !right )
		{
			int L = t4_min( o.readStart, o.seqStart ) ;
			av = t4_overhang_align( pw + 4 * ( o.seqStart - L ), r + o.readStart - L, L, bits + 32 * i, ds ) ;
		}
		else
		{
			int R = t4_min( len - 1 - o.readEnd, seq->len - 1 - o.seqEnd ) ;
			av = t4_overhang_align( pw + 4 * ( o.seqEnd + 1 ), r + o.readEnd + 1, R, bits + 32 * i + 16, ds ) ;
		}
		if ( av.dp )
			t4_count( cx, 1, 1 ) ;
		sstats[x] = t4_side_stats( av, !right ) ;
	}
	T4_SYNC() ;
	T4Ovl *pre = cx.P<T4Ovl>( st->extOff ) ;
	T4_PAR_FOR( i, overlapCnt )
	{
		T4Ovl e ;
		int ok = t4_extend_finish( cx, len, t4_seq( cx, overlaps[i].seqIdx ), factor, overlaps[i], e, sstats[2 * i], sstats[2 * i + 1] ) ;
		e.infoFromHits = ok ;
		pre[i] = e ;
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
	{
		int i ;
		for ( i = 0 ; i < overlapCnt ; ++i )
			if ( pre[i].infoFromHits == 1 && pre[i].readStart == 0 && pre[i].readEnd == len - 1 )
				break ;
		if ( i < overlapCnt )
		{
			sm->e0 = pre[i] ;
			sm->bi[0] = pre[i].seqIdx ;
		}
		else
			sm->bi[0] = -1 ;
		t4_count( cx, 16, (u64)overlapCnt ) ;
	}
	T4_SYNC() ;
	const int ret = sm->bi[0] ;
	T4_SYNC() ;
	return ret ;
}

// A worker's T4Stream is a shell: its own scratch (hit keys, lookup records, overlap arrays, DP rows, slab) plus a copy
// of the set-describing fields of the set it currently serves.  Nothing of the set is written during the launch.
T4_D inline void c_assign_attach( T4Ctx &cx, const T4Stream *set )
{
	T4_SYNC() ;
	if ( cx.tid == 0 )
	{
		T4Stream *st = cx.st ;
		st->kmerLength = set->kmerLength ;
		st->radius = set->radius ;
		st->hitLenRequired = set->hitLenRequired ;
		st->nomatchGapLimit = set->nomatchGapLimit ;
		st->isLongSeqSet = set->isLongSeqSet ;
		st->considerBarcode = set->considerBarcode ;
		st->novelSeqSimilarity = set->novelSeqSimilarity ;
		st->repeatSimilarity = set->repeatSimilarity ;
		st->nSeqs = set->nSeqs ;
		st->seqCap = set->seqCap ;
		st->seqsOff = set->seqsOff ;
		st->dirOff = set->dirOff ;
		st->dirCap = set->dirCap ;
		st->dirUsed = set->dirUsed ;
	}
	T4_SYNC() ;
}

T4_D inline void c_assign_loop( T4Ctx &cx, T4Op *op )
{
	const T4AssignParams *P = t4_x<T4AssignParams>( op->out ) ;
	T4Smem *sm = cx.sm ;
	const int32_t *list = t4_x<int32_t>( P->list ), *leader = t4_x<int32_t>( P->leader ) ;
	const u32 *slotSet = t4_x<u32>( P->slotSet ) ;
	const t4_read_desc *descs = t4_x<t4_read_desc>( P->descs ) ;
	const char *pool = t4_x<char>( P->pool ) ;
	const int8_t *strands = t4_x<int8_t>( P->strands ) ;
	const i64 *descOff = t4_x<i64>( P->descOff ) ;
	int32_t *assign = t4_x<int32_t>( P->assign ) ;
	double *sim = t4_x<double>( P->sim ) ;
	u64 *cursor = t4_x<u64>( P->cursor ) ;
	int cur = -1 ;
	u64 nAssigned = 0 ;
	bool failed = false ;
	while ( 1 )
	{
		T4_SYNC() ;
		if ( cx.tid == 0 )
			sm->bu[0] = t4_atomic_add( cursor, (u64)T4_ASSIGN_CHUNK ) ;
		T4_SYNC() ;
		const i64 c0 = (i64)sm->bu[0] ;
		if ( c0 >= P->nDescs )
			break ;
		const i64 c1 = c0 + T4_ASSIGN_CHUNK < P->nDescs ? c0 + T4_ASSIGN_CHUNK : P->nDescs ;
		for ( i64 s = c0 ; s < c1 ; ++s )
		{
			const int rec = list[s] ;
			if ( rec < 0 || leader[s] != (int32_t)s )
				continue ;
			const int j = (int)slotSet[s] ;
			if ( j != cur )
			{
				c_assign_attach( cx, cx.P<T4Stream>( t4_x<u64>( P->extOff )[j] ) ) ;
				cur = j ;
			}
			const t4_read_desc d = descs[rec] ;
			c_load_read( cx, pool + d.seq_off, d.len ) ;
			const int ret = c_assign_read( cx, d.len, strands[rec], d.barcode ) ;
			failed = c_uniform_error( cx ) != 0 ;
			if ( failed )
				break ;
			// the result goes to this record and to the neighbours that share it (a contiguous range of slots)
			const T4Ovl e = sm->e0 ;
			const i64 hi = descOff[j + 1] ;
			for ( i64 p = s + cx.tid ; p < hi && leader[p] == (int32_t)s ; p += cx.nt )
			{
				int32_t *o = assign + 8 * (i64)list[p] ;
				if ( ret >= 0 )
				{
					o[1] = e.readStart ; o[2] = e.readEnd ; o[3] = e.seqStart ; o[4] = e.seqEnd ;
					o[5] = e.strand ; o[6] = e.matchCnt ; o[7] = 0 ;
					sim[ list[p] ] = e.similarity ;
					o[0] = e.seqIdx ;
					++nAssigned ;
				}
				else
					o[0] = -1 ;
			}
		}
		if ( failed )
			break ;
	}
	T4_SYNC() ;
	if ( nAssigned )
		t4_atomic_add( cursor + 2, nAssigned ) ;
	if ( cx.tid == 0 )
		op->ret = cx.st->error ? cx.st->error : 0 ;
}

// ---- RECOMPUTE ---------------------------------------------------------------------------------------------------
// void SeqSet::RecomputePosWeight( reads ), SeqSet.hpp:4705-4737 (UpdatePosWeightFromRead :2466): zero every column,
// count every assigned read base at seqStart + i (reverse-complemented when the assignment is on strand -1), then give
// the still-empty non-N columns one count of their consensus base.
T4_D inline void c_assign_recompute( T4Ctx &cx, T4Op *op )
{
	const T4AssignParams *P = t4_x<T4AssignParams>( op->out ) ;
	T4Stream *st = cx.st ;
	const int j = op->n ;
	if ( cx.tid == 0 )
		st->novelSeqSimilarity = 0.9 ; // main.cpp:2117
	const int nSeqs = st->nSeqs ;
	for ( int s = 0 ; s < nSeqs ; ++s )
	{
		T4Contig *c = t4_seq( cx, s ) ;
		if ( c->consOff == 0 )
			continue ;
		int *pw = t4_pw( cx, c ) ;
		T4_PAR_FOR( i, 4 * c->len )
			pw[i] = 0 ;
	}
	T4_SYNC() ;
	const i64 lo = t4_x<i64>( P->descOff )[j] ;
	const int cnt = (int)t4_x<u32>( P->listCnt )[j] ;
	const int32_t *list = t4_x<int32_t>( P->list ) ;
	const int32_t *assign = t4_x<int32_t>( P->assign ) ;
	const t4_read_desc *descs = t4_x<t4_read_desc>( P->descs ) ;
	const char *pool = t4_x<char>( P->pool ) ;
	T4_PAR_FOR( p, cnt )
	{
		const int rec = list[lo + p] ;
		const int32_t *a = assign + 8 * (i64)rec ;
		if ( a[0] < 0 )
			continue ;
		T4Contig *c = t4_seq( cx, a[0] ) ;
		u32 *pw = (u32 *)t4_pw( cx, c ) ;
		const t4_read_desc &d = descs[rec] ;
		const char *rd = pool + d.seq_off ;
		const int seqStart = a[3] ;
		for ( int i = 0 ; i < d.len ; ++i )
		{
			char ch ;
			if ( a[5] == 1 )
				ch = rd[i] ;
			else
			{
				const char f = rd[d.len - 1 - i] ;
				ch = ( f != 'N' ) ? t4_numToNuc( 3 - t4_nuc( f ) ) : 'N' ;
			}
			if ( ch != 'N' && seqStart + i >= 0 && seqStart + i < c->len )
				t4_atomic_add32( pw + 4 * ( seqStart + i ) + t4_nuc( ch ), 1u ) ;
		}
	}
	T4_SYNC() ;
	for ( int s = 0 ; s < nSeqs ; ++s )
	{
		T4Contig *c = t4_seq( cx, s ) ;
		if ( c->consOff == 0 )
			continue ;
		int *pw = t4_pw( cx, c ) ;
		unsigned char *eq = t4_eq( cx, c ) ;
		const char *cons = t4_cons( cx, c ) ;
		// the counts were zeroed and added with atomics above: every column's equality byte is refreshed here, once
		// they are final
		T4_PAR_FOR( i, c->len )
		{
			if ( cons[i] != 'N' && pw[4 * i] + pw[4 * i + 1] + pw[4 * i + 2] + pw[4 * i + 3] == 0 )
				t4_col_add( pw, eq, i, t4_nuc( cons[i] ), 1 ) ;
			else
				eq[i] = (unsigned char)t4_eq_nibble( pw + 4 * i ) ;
		}
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
		op->ret = 0 ;
}

// ---- dispatch: body of the auxiliary kernel (one CTA = one T4Op) ----------------------------------------------------
T4_D inline void c_run_aux_op_more( T4Ctx &cx, T4Op *op ) ; // t4_refscan.h: the reference-set ops

T4_D inline void c_run_aux_op( T4Ctx &cx, T4Op *op )
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
	if ( cx.st->error )
	{
		if ( cx.tid == 0 )
			op->ret = cx.st->error ;
		return ;
	}
	switch ( op->op )
	{
		case T4_OP_ASSIGN_PREP:
			c_assign_prep( cx, op ) ;
			break ;
		case T4_OP_ASSIGN:
			c_assign_loop( cx, op ) ;
			break ;
		case T4_OP_GROUP_HITS:
			c_test_group_hits( cx, op ) ;
			break ;
		case T4_OP_ASSIGN_RECOMPUTE:
			c_assign_recompute( cx, op ) ;
			break ;
		default:
			c_run_aux_op_more( cx, op ) ;
			break ;
	}
	T4_SYNC() ;
	if ( cx.tid == 0 && cx.st->error && op->ret >= T4_E_BASE )
		op->ret = cx.st->error ;
	if ( cx.tid == 0 )
		for ( int i = 0 ; i < T4_N_COUNTERS ; ++i )
			if ( ( i < 8 || i >= 16 ) && sm->ctr[i] )
				t4_atomic_add( &cx.g->counters[i], sm->ctr[i] ) ;
#if T4_CUDA
	T4_PHASE( cx, 0 ) ;
	if ( cx.tid == 0 )
	{
		u64 tot = 0 ;
		for ( int i = 0 ; i < 8 ; ++i )
			tot += (u64)sm->ph[i] ;
		cx.st->nReads = tot ; // clock cycles of this op on this CTA (t4_streams_cycles)
	}
#endif
}

#endif
