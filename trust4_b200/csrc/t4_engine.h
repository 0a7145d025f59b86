// Stream engine: the per-read k-mer-seeded overlap-and-extend assembly hot path
// (KmerIndex lookup -> hit chaining -> banded DP extension -> posWeight update)
// as device code executed by ONE CTA PER STREAM (= per SeqSet).
//
// Written against T4Ctx{tid, nt} + T4_SYNC(): compiled by nvcc for sm_90a
// (product) and by g++ with nt = 1 for the test-only emulation (tests/emu).
// Function prefixes:  c_  collective (every thread of the CTA calls it; contains
// barriers),  s_  serial (thread 0 only),  no prefix: pure / any thread.
//
// Every function cites the reference code whose observable behaviour it
// reproduces (paths relative to the reference tree).  This is a re-design, not a
// translation: hits are single 64-bit keys sorted by a CTA radix sort, chains are
// diagonal runs of the sorted key array, contigs live in slack-padded HBM arrays
// so a left extension is a pointer move, postings are unordered multisets
// (their order is unobservable: GetOverlapsFromHits re-sorts every group).
#ifndef T4_ENGINE_H
#define T4_ENGINE_H

#include "t4_common.h"

#if !T4_CUDA
#include <algorithm>
#endif

#define T4_MAX_NT 128
#define T4_IDX_CHUNK 256
#define T4_WACT_WORDS 12
#define T4_SMEM_SORT ( T4_RADIX * T4_MAX_NT / 2 )
#define T4_RADIX_BITS 4
#define T4_RADIX (1 << T4_RADIX_BITS)
#define T4_DP_BAND 5
#define T4_DP_W (2 * T4_DP_BAND + 3)

#define EDIT_MATCH 0
#define EDIT_MISMATCH 1
#define EDIT_INSERT 2
#define EDIT_DELETE 3
#define SCORE_MATCH 2
#define SCORE_MISMATCH (-2)
#define SCORE_INDEL (-4)

// What AddRead's decision walk and merge commit (thread 0) hand its collective phases (c_add_read).  kind: 0 nothing
// to commit, 1 extend / inside the contig of e0, 2 merged (the merge is done).  AssignRead's result is e0 as well.
struct T4AddPlan
{
	T4Ovl e0 ;
	int kind ;
	int seqIdx ;
	int readInConsensusOffset ;
	int ret ;
	bool bail ;
	bool added ;
} ;

struct T4Smem
{
	char read[T4_DEV_MAX_READ + 8] ;
	char rc[T4_DEV_MAX_READ + 8] ;
	u32 radix[T4_RADIX * T4_MAX_NT] ;
	u32 scan[T4_MAX_NT + 4] ;
	u64 bu[4] ;
	int bi[16] ;
	u64 red[2] ;
	u64 icode[T4_IDX_CHUNK] ; // c_index_op: k-mer codes of the current chunk of positions
	unsigned char iact[T4_IDX_CHUNK] ;
	T4AddPlan plan ;
	u32 wnib[T4_MAX_NT / 32][2][64] ;        // per warp, per overhang side: IsBaseEqual nibbles of up to 512 columns
	u32 wbits[T4_MAX_NT / 32][2][16] ;       // ... and the match bits against the read
	u32 wact[T4_MAX_NT / 32][2][13 * T4_WACT_WORDS] ; // ... traceback words of the half-warp DP (n <= 16*T4_WACT_WORDS - 1)
	signed char wal[T4_MAX_NT / 32][2][2 * 16 * T4_WACT_WORDS + 8] ; // ... and its edit string (filled backwards: no reversal pass)
	u64 ctr[T4_N_COUNTERS] ; // device counters of this op, flushed to the arena header once at the end
	long long ph[8] ;      // per-phase clock accumulators (thread 0)
	long long phLast ;
	int phCur ;
} ;

struct T4Ctx
{
	char *A ;          // arena base
	T4Global *g ;
	T4Stream *st ;
	T4Smem *sm ;
	u64 cap ;          // arena capacity (copy of g->cap)
	int tid, nt ;

	template <class T> T4_HD T *P( u64 off ) const { return (T *)( A + off ) ; }
} ;

// The context of thread tid of nt working on the stream at arena offset streamOff.
T4_HD inline T4Ctx t4_ctx( char *A, u64 streamOff, T4Smem *sm, int tid, int nt )
{
	T4Ctx cx ;
	cx.A = A ;
	cx.g = (T4Global *)A ;
	cx.st = (T4Stream *)( A + streamOff ) ;
	cx.sm = sm ;
	cx.cap = cx.g->cap ;
	cx.tid = tid ;
	cx.nt = nt ;
	return cx ;
}

#define T4_PAR_FOR( i, n ) for ( int i = cx.tid ; i < (int)( n ) ; i += cx.nt )

T4_D inline u64 t4_atomic_cas( u64 *p, u64 cmp, u64 val ) ;

T4_D inline void t4_raise( T4Ctx &cx, int code, int aux )
{
	if ( cx.st->error == 0 )
	{
		cx.st->error = code ;
		cx.st->errorAux = aux ;
	}
	if ( cx.g->firstError == 0 )
		t4_atomic_cas( &cx.g->firstError, 0ull, (u64)(u32)code | ( (u64)(u32)aux << 32 ) ) ;
}

T4_D inline void t4_count( T4Ctx &cx, int idx, u64 v )
{
	if ( v == 0 )
		return ;
#if T4_CUDA
	atomicAdd( (unsigned long long *)&cx.sm->ctr[idx], (unsigned long long)v ) ;
#else
	cx.sm->ctr[idx] += v ;
#endif
}

// phase accounting (thread 0): 0 other, 1 probe, 2 hit sort, 3 chains, 4 overlap sort + scoring, 5 ExtendOverlap,
// 6 decision + commit, 7 InputNovelRead / RepeatAddRead / consensus maintenance
#if T4_CUDA
#define T4_PHASE( cx, id )                                       \
	do                                                           \
	{                                                            \
		if ( ( cx ).tid == 0 )                                   \
		{                                                        \
			long long now_ = clock64() ;                         \
			( cx ).sm->ph[( cx ).sm->phCur] += now_ - ( cx ).sm->phLast ; \
			( cx ).sm->phLast = now_ ;                           \
			( cx ).sm->phCur = ( id ) ;                          \
		}                                                        \
	} while ( 0 )
#else
#define T4_PHASE( cx, id ) ( (void)0 )
#endif

// ---------------------------------------------------------------------------
// small utilities
// ---------------------------------------------------------------------------
T4_HD inline int t4_nuc( char c ) // nucToNum[c - 'A'] & 3 (main.cpp:39-42): A0 C1 G2 T3, N -> 0, anything else -> 3
{
	// two bits per letter 'A' .. 'Z' in one constant: as a switch this is a jump table, and the lanes of a warp, which
	// hold different bases, take its branches one after the other
	const unsigned d = (unsigned)(unsigned char)c - 'A' ;
	return d < 26u ? (int)( ( 0xffffff3ffefdcull >> ( 2 * d ) ) & 3u ) : 3 ;
}
T4_HD inline char t4_numToNuc( int x ) { return "ACGT"[x & 3] ; }

T4_HD inline int t4_abs( int x ) { return x < 0 ? -x : x ; }
T4_HD inline int t4_min( int a, int b ) { return a < b ? a : b ; }
T4_HD inline int t4_max( int a, int b ) { return a > b ? a : b ; }

T4_D inline u64 t4_atomic_add( u64 *p, u64 v )
{
#if T4_CUDA
	return atomicAdd( (unsigned long long *)p, (unsigned long long)v ) ;
#else
	u64 o = *p ; *p += v ; return o ;
#endif
}

T4_D inline u64 t4_atomic_cas( u64 *p, u64 cmp, u64 val )
{
#if T4_CUDA
	return atomicCAS( (unsigned long long *)p, (unsigned long long)cmp, (unsigned long long)val ) ;
#else
	u64 o = *p ;
	if ( o == cmp )
		*p = val ;
	return o ;
#endif
}

T4_D inline u32 t4_atomic_add32( u32 *p, u32 v )
{
#if T4_CUDA
	return atomicAdd( p, v ) ;
#else
	u32 o = *p ; *p += v ; return o ;
#endif
}

struct T4Ctx ;
T4_D inline void t4_count( T4Ctx &cx, int idx, u64 v ) ;

T4_D inline void t4_raise( T4Ctx &cx, int code, int aux ) ;

// Bump allocation from the arena; callable by any thread.  Returns 0 (and raises T4_E_NOMEM) when exhausted.
// Small requests are served from a stream-local slab (refilled by thread 0 between reads, c_refill_slab) so
// that thousands of CTAs do not serialise on the one global bump pointer.
#define T4_SLAB_BYTES ( 128u << 10 )
#define T4_SLAB_MAX_REQ ( 8u << 10 )

T4_D inline u64 t4_alloc_global( T4Ctx &cx, u64 bytes )
{
	u64 off = t4_atomic_add( &cx.g->top, bytes ) ;
	if ( off + bytes > cx.cap )
	{
		t4_raise( cx, T4_E_NOMEM, (int)( bytes >> 10 ) ) ;
		return 0 ;
	}
	return off ;
}

T4_D inline u64 s_alloc( T4Ctx &cx, u64 bytes )
{
	bytes = ( bytes + ( T4_ALIGN - 1 ) ) & ~(u64)( T4_ALIGN - 1 ) ;
	T4Stream *st = cx.st ;
	if ( st != 0 && bytes <= T4_SLAB_MAX_REQ && st->slabTop + bytes <= st->slabEnd )
	{
		u64 off = t4_atomic_add( &st->slabTop, bytes ) ;
		if ( off + bytes <= st->slabEnd )
			return off ;
	}
	return t4_alloc_global( cx, bytes ) ;
}

// Thread 0, at a point where no other thread allocates: start a fresh slab when the current one runs low.
T4_D inline void s_refill_slab( T4Ctx &cx )
{
	T4Stream *st = cx.st ;
	if ( st->slabTop + ( T4_SLAB_BYTES / 4 ) > st->slabEnd )
	{
		u64 off = t4_alloc_global( cx, T4_SLAB_BYTES ) ;
		if ( off )
		{
			st->slabTop = off ;
			st->slabEnd = off + T4_SLAB_BYTES ;
		}
	}
}

T4_D inline T4Contig *t4_seq( T4Ctx &cx, int idx ) { return cx.P<T4Contig>( cx.st->seqsOff ) + idx ; }
T4_D inline char *t4_cons( T4Ctx &cx, T4Contig *c ) { return cx.P<char>( c->consOff ) + c->lead ; }
T4_D inline int *t4_pw( T4Ctx &cx, T4Contig *c ) { return cx.P<int>( c->pwOff ) + 4 * c->lead ; }
// Equality byte of every posWeight column, stored behind the posWeight array of the same allocation (so T4Contig stays
// two sectors and no contig can have counts without bytes): bit b set iff AlignAlgo::IsBaseEqual( column, base b )
// (AlignAlgo.hpp:49-55, an 'N' read base matches everything at the consumer).  The overhang masks, the gap scoring and
// the overhang DPs read one byte per column instead of four counts.
T4_D inline unsigned char *t4_eq( T4Ctx &cx, T4Contig *c ) { return cx.P<unsigned char>( c->pwOff + 16ull * c->cap ) + c->lead ; }
#define T4_PW_BYTES( cap ) ( (u64)( cap ) * 17 )

T4_HD inline unsigned t4_eq_nibble( const int *w )
{
	int sum = w[0] + w[1] + w[2] + w[3] ;
	if ( sum == 0 )
		return 0xFu ;
	return ( sum < 3 * w[0] ? 1u : 0u ) | ( sum < 3 * w[1] ? 2u : 0u ) | ( sum < 3 * w[2] ? 4u : 0u ) | ( sum < 3 * w[3] ? 8u : 0u ) ;
}

// Every store of posWeight counts goes through these two (or copies a column together with its byte), so the equality
// byte stays a function of the column.  Column col of pw / eq (both from the contig's lead).
T4_HD inline void t4_col_put( int *pw, unsigned char *eq, int col, int a, int c, int g, int t )
{
	int *w = pw + 4 * col ;
	w[0] = a ; w[1] = c ; w[2] = g ; w[3] = t ;
	eq[col] = (unsigned char)t4_eq_nibble( w ) ;
}
T4_HD inline void t4_col_add( int *pw, unsigned char *eq, int col, int b, int d )
{
	int *w = pw + 4 * col ;
	w[b] += d ;
	eq[col] = (unsigned char)t4_eq_nibble( w ) ;
}

T4_D inline u64 t4_key_of( int strand, int idx, int a, int b, int bigRepeat )
{
	return ( (u64)( strand == 1 ? 1 : 0 ) << T4_KEY_STRAND_SHIFT ) | ( (u64)(u32)idx << T4_KEY_IDX_SHIFT )
		| ( (u64)(u32)( a - b + T4_KEY_C_BIAS ) << T4_KEY_C_SHIFT ) | ( (u64)(u32)b << T4_KEY_B_SHIFT ) | (u64)( bigRepeat ? 1 : 0 ) ;
}
T4_HD inline int t4_key_strand( u64 k ) { return ( k >> T4_KEY_STRAND_SHIFT ) ? 1 : -1 ; }
T4_HD inline int t4_key_idx( u64 k ) { return (int)( ( k >> T4_KEY_IDX_SHIFT ) & ( ( 1u << T4_KEY_IDX_BITS ) - 1 ) ) ; }
T4_HD inline int t4_key_b( u64 k ) { return (int)( ( k >> T4_KEY_B_SHIFT ) & T4_KEY_B_MASK ) ; }
T4_HD inline int t4_key_c( u64 k ) { return (int)( ( k >> T4_KEY_C_SHIFT ) & T4_KEY_C_MASK ) - T4_KEY_C_BIAS ; }
T4_HD inline int t4_key_a( u64 k ) { return t4_key_b( k ) + t4_key_c( k ) ; }
T4_HD inline int t4_key_big( u64 k ) { return (int)( k & 1 ) ; }

// ---------------------------------------------------------------------------
// k-mer directory + postings (KmerIndex.hpp).  Open addressing, 32-byte slots.
// ---------------------------------------------------------------------------
T4_D inline u64 t4_index_key( T4Stream *st, u64 code, int barcode )
{
	// KmerIndex::GetHash salts the bucket with barcode + 1 when considerBarcode is set (KmerIndex.hpp:29-33): bucket
	// (code + barcode + 1) % 1000003, and inside the bucket the map key is the code alone.  So one postings list serves
	// every barcode of one residue (barcode + 1) % 1000003: barcodes 5 and 1000008 share their lists, barcode -1 shares
	// with 1000002.  The salt is that residue; the barcode filter of GetHitsFromRead drops the foreign postings.
	u64 key = code ;
	if ( st->considerBarcode )
		key += (u64)( (u32)( barcode + 1 ) % T4_KINDEX_HASH_MAX ) << ( 2 * st->kmerLength ) ;
	return key + 1 ;
}

// Load factor of the directory stays <= 1 / T4_DIR_INV_LOAD.  1/4: an absent k-mer (most probes of a read are misses)
// then needs 1.4 slot reads on average instead of 2.5 at 1/2, and a warp waits for the longest chain among its lanes.
#define T4_DIR_INV_LOAD 4
T4_D inline u32 t4_dir_slot( u64 key, u32 cap ) { return (u32)( ( key * 0x9E3779B97F4A7C15ull ) >> 32 ) & ( cap - 1 ) ; }

T4_D inline T4Dir *t4_dir_find( T4Ctx &cx, u64 key )
{
	T4Stream *st = cx.st ;
	T4Dir *dir = cx.P<T4Dir>( st->dirOff ) ;
	u32 cap = st->dirCap ;
	u32 s = t4_dir_slot( key, cap ) ;
	while ( 1 )
	{
		u64 kk = dir[s].key ;
		if ( kk == key )
			return dir + s ;
		if ( kk == 0 )
			return 0 ;
		s = ( s + 1 ) & ( cap - 1 ) ;
	}
}

T4_D inline void s_dir_grow( T4Ctx &cx )
{
	T4Stream *st = cx.st ;
	u32 oldCap = st->dirCap ;
	u32 newCap = oldCap * 2 ;
	u64 off = s_alloc( cx, (u64)newCap * sizeof( T4Dir ) ) ;
	if ( !off )
		return ;
	T4Dir *nd = cx.P<T4Dir>( off ) ;
	T4Dir *od = cx.P<T4Dir>( st->dirOff ) ;
	for ( u32 i = 0 ; i < newCap ; ++i )
		nd[i].key = 0 ;
	for ( u32 i = 0 ; i < oldCap ; ++i )
	{
		if ( od[i].key == 0 )
			continue ;
		u32 s = t4_dir_slot( od[i].key, newCap ) ;
		while ( nd[s].key != 0 )
			s = ( s + 1 ) & ( newCap - 1 ) ;
		nd[s] = od[i] ;
	}
	st->dirOff = off ;
	st->dirCap = newCap ;
}

// Collective variant: zero and re-insert in parallel (keys are unique, slots are claimed with a CAS).
T4_D inline void c_dir_grow( T4Ctx &cx )
{
	T4Stream *st = cx.st ;
	T4_SYNC() ;
	u32 oldCap = st->dirCap ;
	u32 newCap = oldCap * 2 ;
	if ( cx.tid == 0 )
	{
		u64 off = s_alloc( cx, (u64)newCap * sizeof( T4Dir ) ) ;
		cx.sm->bu[0] = off ;
	}
	T4_SYNC() ;
	u64 off = cx.sm->bu[0] ;
	T4_SYNC() ;
	if ( !off )
		return ;
	T4Dir *nd = cx.P<T4Dir>( off ) ;
	T4Dir *od = cx.P<T4Dir>( st->dirOff ) ;
	for ( u32 i = cx.tid ; i < newCap ; i += cx.nt )
		nd[i].key = 0 ;
	T4_SYNC() ;
	for ( u32 i = cx.tid ; i < oldCap ; i += cx.nt )
	{
		T4Dir e = od[i] ;
		if ( e.key == 0 )
			continue ;
		u32 s = t4_dir_slot( e.key, newCap ) ;
		while ( 1 )
		{
			if ( nd[s].key == 0 && t4_atomic_cas( &nd[s].key, 0ull, e.key ) == 0 )
				break ;
			s = ( s + 1 ) & ( newCap - 1 ) ;
		}
		nd[s].listOff = e.listOff ;
		nd[s].cnt = e.cnt ;
		nd[s].cap = e.cap ;
		nd[s].lock = 0 ;
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
	{
		st->dirOff = off ;
		st->dirCap = newCap ;
	}
	T4_SYNC() ;
}

T4_D inline T4Dir *s_dir_get( T4Ctx &cx, u64 key )
{
	T4Stream *st = cx.st ;
	if ( ( st->dirUsed + 1 ) * T4_DIR_INV_LOAD > st->dirCap )
	{
		s_dir_grow( cx ) ;
		if ( st->error )
			return 0 ;
	}
	T4Dir *dir = cx.P<T4Dir>( st->dirOff ) ;
	u32 cap = st->dirCap ;
	u32 s = t4_dir_slot( key, cap ) ;
	while ( 1 )
	{
		u64 kk = dir[s].key ;
		if ( kk == key )
			return dir + s ;
		if ( kk == 0 )
		{
			dir[s].key = key ;
			dir[s].listOff = 0 ;
			dir[s].cnt = 0 ;
			dir[s].cap = 0 ;
			dir[s].lock = 0 ;
			++st->dirUsed ;
			return dir + s ;
		}
		s = ( s + 1 ) & ( cap - 1 ) ;
	}
}

// KmerIndex::Insert (KmerIndex.hpp:66).  Postings are an unordered multiset.
T4_D inline void s_index_insert( T4Ctx &cx, u64 code, int idx, int offset, int barcode )
{
	T4Dir *d = s_dir_get( cx, t4_index_key( cx.st, code, barcode ) ) ;
	if ( !d )
		return ;
	if ( d->cnt == d->cap )
	{
		u32 nc = d->cap ? d->cap * 2 : 4 ;
		u64 off = s_alloc( cx, (u64)nc * 8 ) ;
		if ( !off )
			return ;
		u64 *nl = cx.P<u64>( off ) ;
		u64 *ol = cx.P<u64>( d->listOff ) ;
		for ( u32 i = 0 ; i < d->cnt ; ++i )
			nl[i] = ol[i] ;
		d->listOff = off ;
		d->cap = nc ;
	}
	cx.P<u64>( d->listOff )[d->cnt] = ( (u64)(u32)idx << 32 ) | (u32)offset ;
	++d->cnt ;
}

// KmerIndex::Remove (KmerIndex.hpp:81): delete one posting equal to (idx, offset) if present.
T4_D inline void s_index_remove( T4Ctx &cx, u64 code, int idx, int offset, int barcode )
{
	T4Dir *d = t4_dir_find( cx, t4_index_key( cx.st, code, barcode ) ) ;
	if ( !d )
		return ;
	u64 v = ( (u64)(u32)idx << 32 ) | (u32)offset ;
	u64 *l = cx.P<u64>( d->listOff ) ;
	for ( u32 i = 0 ; i < d->cnt ; ++i )
		if ( l[i] == v )
		{
			l[i] = l[d->cnt - 1] ;
			--d->cnt ;
			return ;
		}
}

// Rolling 2-bit k-mer with N tracking (KmerCode.hpp:94-109).
struct T4Kmer
{
	u64 code, mask ;
	int k, sinceN ;    // sinceN: bases appended since the last 'N' (saturating), valid iff >= k
	T4_D inline void init( int kl )
	{
		k = kl ;
		mask = kl < 32 ? ( ( 1ull << ( 2 * kl ) ) - 1ull ) : ~0ull ;
		code = 0 ;
		sinceN = 1 << 20 ;
	}
	T4_D inline void restart() { code = 0 ; sinceN = 1 << 20 ; }
	T4_D inline void append( char c )
	{
		code = ( ( code << 2 ) & mask ) | (u64)t4_nuc( c ) ;
		if ( c == 'N' )
			sinceN = 0 ;
		else if ( sinceN < ( 1 << 20 ) )
			++sinceN ;
	}
	T4_D inline bool valid() const { return sinceN >= k ; }
} ;

// KmerIndex::BuildIndexFromRead (KmerIndex.hpp:118-141), including its first-k-mer rule (i == kl, not kl-1).
T4_D inline void s_build_index( T4Ctx &cx, const char *s, int len, int id, int barcode, int shift )
{
	int kl = cx.st->kmerLength ;
	if ( len < kl )
		return ;
	T4Kmer km ;
	km.init( kl ) ;
	u64 prev = 0 ;
	int i ;
	for ( i = 0 ; i < kl - 1 ; ++i )
		km.append( s[i] ) ;
	for ( ; i < len ; ++i )
	{
		km.append( s[i] ) ;
		if ( km.valid() && ( i == kl || km.code != prev ) )
			s_index_insert( cx, km.code, id, i - kl + 1 + shift, barcode ) ;
		prev = km.code ;
	}
}

// KmerIndex::UpdateIndexFromRead (KmerIndex.hpp:144-181): literal, position by position.
T4_D inline void s_update_index( T4Ctx &cx, const char *s, int len, int barcode, int shift, int oldId, int id )
{
	int kl = cx.st->kmerLength ;
	if ( len < kl )
		return ;
	T4Kmer km ;
	km.init( kl ) ;
	int i ;
	for ( i = 0 ; i < kl - 1 ; ++i )
		km.append( s[i] ) ;
	for ( ; i < len ; ++i )
	{
		km.append( s[i] ) ;
		if ( !km.valid() )
			continue ;
		T4Dir *d = t4_dir_find( cx, t4_index_key( cx.st, km.code, barcode ) ) ;
		if ( !d )
			continue ;
		u64 v = ( (u64)(u32)oldId << 32 ) | (u32)( i - kl + 1 ) ;
		u64 *l = cx.P<u64>( d->listOff ) ;
		for ( u32 j = 0 ; j < d->cnt ; ++j )
			if ( l[j] == v )
			{
				l[j] = ( (u64)(u32)id << 32 ) | (u32)( i - kl + 1 + shift ) ;
				break ;
			}
	}
}

// KmerIndex::RemoveIndexFromRead (KmerIndex.hpp:183-201).
T4_D inline void s_remove_index( T4Ctx &cx, const char *s, int len, int id, int barcode, int offset )
{
	int kl = cx.st->kmerLength ;
	if ( len < kl )
		return ;
	T4Kmer km ;
	km.init( kl ) ;
	int i ;
	for ( i = 0 ; i < kl - 1 ; ++i )
		km.append( s[i] ) ;
	for ( ; i < len ; ++i )
	{
		km.append( s[i] ) ;
		if ( km.valid() )
			s_index_remove( cx, km.code, id, i - kl + 1 + offset, barcode ) ;
	}
}

// ---------------------------------------------------------------------------
// collective index maintenance.  The three KmerIndex walkers (Build / Update / RemoveIndexFromRead,
// KmerIndex.hpp:118-201) only interact through the postings list of ONE k-mer code, so positions are
// processed in chunks, every distinct code of a chunk is owned by the thread of its first occurrence,
// and the owner applies that code's positions in ascending order -- exactly the reference's sequence
// restricted to that list.  Chunks run one after the other, so order across chunks is ascending too.
// ---------------------------------------------------------------------------
T4_D inline u32 c_scan_threads( T4Ctx &cx, u32 v, u32 &total ) ;

#define T4_IDX_BUILD 0
#define T4_IDX_REMOVE 1
#define T4_IDX_UPDATE 2

T4_D inline T4Dir *t4_dir_find_or_claim( T4Ctx &cx, u64 key )
{
	T4Stream *st = cx.st ;
	T4Dir *dir = cx.P<T4Dir>( st->dirOff ) ;
	u32 cap = st->dirCap ;
	u32 s = t4_dir_slot( key, cap ) ;
	while ( 1 )
	{
		u64 kk = dir[s].key ;
		if ( kk == key )
			return dir + s ;
		if ( kk == 0 )
		{
			u64 old = t4_atomic_cas( &dir[s].key, 0ull, key ) ;
			if ( old == 0 )
			{
				dir[s].listOff = 0 ;
				dir[s].cnt = 0 ;
				dir[s].cap = 0 ;
				dir[s].lock = 0 ;
				t4_atomic_add32( &st->dirUsed, 1 ) ;
				return dir + s ;
			}
			if ( old == key )
				return dir + s ;
		}
		s = ( s + 1 ) & ( cap - 1 ) ;
	}
}

T4_D inline void t4_list_append( T4Ctx &cx, T4Dir *d, u64 v )
{
	if ( d->cnt == d->cap )
	{
		u32 nc = d->cap ? d->cap * 2 : 4 ;
		u64 off = s_alloc( cx, (u64)nc * 8 ) ;
		if ( !off )
			return ;
		u64 *nl = cx.P<u64>( off ) ;
		u64 *ol = cx.P<u64>( d->listOff ) ;
		for ( u32 i = 0 ; i < d->cnt ; ++i )
			nl[i] = ol[i] ;
		d->listOff = off ;
		d->cap = nc ;
	}
	cx.P<u64>( d->listOff )[d->cnt] = v ;
	++d->cnt ;
}

// mode BUILD:  BuildIndexFromRead( s, len, id, barcode, shift = arg )
// mode REMOVE: RemoveIndexFromRead( s, len, id, barcode, offset = arg )
// mode UPDATE: UpdateIndexFromRead( s, len, barcode, shift = arg, oldId, id )
T4_D T4_BIG void c_index_op( T4Ctx &cx, const char *s, int len, int mode, int id, int barcode, int arg, int oldId )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	const int kl = st->kmerLength ;
	T4_SYNC() ;
	if ( len < kl )
		return ;
	const u64 mask = kl < 32 ? ( ( 1ull << ( 2 * kl ) ) - 1ull ) : ~0ull ;
	for ( int c0 = kl - 1 ; c0 < len ; c0 += T4_IDX_CHUNK )
	{
		int cn = len - c0 < T4_IDX_CHUNK ? len - c0 : T4_IDX_CHUNK ;
		u32 mine = 0 ;
		T4_PAR_FOR( j, cn )
		{
			int i = c0 + j ;
			u64 code = 0 ;
			bool valid = true ;
			for ( int x = i - kl + 1 ; x <= i ; ++x )
			{
				char c = s[x] ;
				code = ( code << 2 ) | (u64)t4_nuc( c ) ;
				if ( c == 'N' )
					valid = false ;
			}
			bool act = valid ;
			if ( mode == T4_IDX_BUILD && valid )
			{
				u64 prev = 0 ; // KmerCode prevKmerCode( kl ) starts at 0; afterwards the rolling code of position i-1
				if ( i > kl - 1 )
					prev = ( ( code >> 2 ) | ( (u64)t4_nuc( s[i - kl] ) << ( 2 * ( kl - 1 ) ) ) ) & mask ;
				act = ( i == kl || code != prev ) ;
			}
			sm->icode[j] = code ;
			sm->iact[j] = act ? 1 : 0 ;
			if ( act )
				++mine ;
		}
		if ( mode == T4_IDX_BUILD )
		{
			u32 total ;
			c_scan_threads( cx, mine, total ) ;
			while ( !st->error && ( st->dirUsed + total + 1 ) * T4_DIR_INV_LOAD > st->dirCap )
				c_dir_grow( cx ) ;
		}
		T4_SYNC() ;
		if ( st->error )
			return ;
		T4_PAR_FOR( j, cn )
		{
			if ( !sm->iact[j] )
				continue ;
			u64 code = sm->icode[j] ;
			// uniform scan of the chunk (same trip count in every lane, broadcast shared-memory reads)
			int first = -1, nsame = 0 ;
			for ( int x = 0 ; x < cn ; ++x )
				if ( sm->icode[x] == code && sm->iact[x] )
				{
					if ( first < 0 )
						first = x ;
					++nsame ;
				}
			if ( first != j )
				continue ;
			u64 key = t4_index_key( st, code, barcode ) ;
			T4Dir *d = ( mode == T4_IDX_BUILD ) ? t4_dir_find_or_claim( cx, key ) : t4_dir_find( cx, key ) ;
			if ( !d )
				continue ;
			for ( int x = j ; x < cn && nsame > 0 ; ++x )
			{
				if ( !sm->iact[x] || sm->icode[x] != code )
					continue ;
				--nsame ;
				int pos = c0 + x - kl + 1 ;
				if ( mode == T4_IDX_BUILD )
					t4_list_append( cx, d, ( (u64)(u32)id << 32 ) | (u32)( pos + arg ) ) ;
				else if ( mode == T4_IDX_REMOVE )
				{
					u64 v = ( (u64)(u32)id << 32 ) | (u32)( pos + arg ) ;
					u64 *l = cx.P<u64>( d->listOff ) ;
					for ( u32 y = 0 ; y < d->cnt ; ++y )
						if ( l[y] == v )
						{
							l[y] = l[d->cnt - 1] ;
							--d->cnt ;
							break ;
						}
				}
				else
				{
					u64 v = ( (u64)(u32)oldId << 32 ) | (u32)pos ;
					u64 *l = cx.P<u64>( d->listOff ) ;
					for ( u32 y = 0 ; y < d->cnt ; ++y )
						if ( l[y] == v )
						{
							l[y] = ( (u64)(u32)id << 32 ) | (u32)( pos + arg ) ;
							break ;
						}
				}
			}
		}
		T4_SYNC() ;
	}
}

// ---------------------------------------------------------------------------
// contig storage
// ---------------------------------------------------------------------------
// Append a contig slot (seqs.push_back).  Serial.
T4_D inline int s_new_contig( T4Ctx &cx, int len )
{
	T4Stream *st = cx.st ;
	if ( st->nSeqs == st->seqCap )
	{
		int nc = st->seqCap * 2 ;
		u64 off = s_alloc( cx, (u64)nc * sizeof( T4Contig ) ) ;
		if ( !off )
			return -1 ;
		T4Contig *n = cx.P<T4Contig>( off ) ;
		T4Contig *o = cx.P<T4Contig>( st->seqsOff ) ;
		for ( int i = 0 ; i < st->nSeqs ; ++i )
			n[i] = o[i] ;
		st->seqsOff = off ;
		st->seqCap = nc ;
	}
	if ( st->nSeqs >= ( 1 << T4_KEY_IDX_BITS ) - 1 )
	{
		t4_raise( cx, T4_E_UNSUPPORTED, 1 ) ;
		return -1 ;
	}
	int idx = st->nSeqs ;
	T4Contig *c = t4_seq( cx, idx ) ;
	int cap = 2 * len + 128 ;
	c->consOff = s_alloc( cx, cap ) ;
	c->pwOff = s_alloc( cx, T4_PW_BYTES( cap ) ) ;
	if ( !c->consOff || !c->pwOff )
		return -1 ;
	c->cap = cap ;
	c->lead = ( cap - len ) / 2 ;
	c->len = len ;
	c->nameOff = 0 ;
	c->nameLen = 0 ;
	c->minLeftExtAnchor = c->minRightExtAnchor = 0 ;
	c->barcode = -1 ;
	c->numRead = 0 ;
	c->flags = 0 ;
	c->packNarrow = 0 ;
	++st->nSeqs ;
	return idx ;
}

// Make room for `left` new bases in front and `right` behind; old bases keep their values,
// new cells are uninitialised.  Serial.
T4_D inline bool s_contig_grow( T4Ctx &cx, T4Contig *c, int left, int right )
{
	int newLen = c->len + left + right ;
	if ( newLen > (int)T4_KEY_B_MASK )
	{
		t4_raise( cx, T4_E_UNSUPPORTED, 2 ) ;
		return false ;
	}
	if ( c->lead >= left && c->lead + c->len + right <= c->cap )
	{
		c->lead -= left ;
		c->len = newLen ;
		return true ;
	}
	int cap = 2 * newLen + 128 ;
	u64 co = s_alloc( cx, cap ) ;
	u64 po = s_alloc( cx, T4_PW_BYTES( cap ) ) ;
	if ( !co || !po )
		return false ;
	int lead = ( cap - newLen ) / 2 ;
	char *oc = t4_cons( cx, c ) ;
	int *op = t4_pw( cx, c ) ;
	const unsigned char *oe = t4_eq( cx, c ) ;
	char *nc = cx.P<char>( co ) + lead + left ;
	int *np = cx.P<int>( po ) + 4 * ( lead + left ) ;
	unsigned char *ne = cx.P<unsigned char>( po + 16ull * cap ) + lead + left ;
	for ( int i = 0 ; i < c->len ; ++i )
		nc[i] = oc[i] ;
	for ( int i = 0 ; i < 4 * c->len ; ++i )
		np[i] = op[i] ;
	for ( int i = 0 ; i < c->len ; ++i )
		ne[i] = oe[i] ;
	c->consOff = co ;
	c->pwOff = po ;
	c->cap = cap ;
	c->lead = lead ;
	c->len = newLen ;
	return true ;
}

T4_D inline void s_set_name( T4Ctx &cx, T4Contig *c, const char *s, int n )
{
	u64 off = s_alloc( cx, n + 1 ) ;
	if ( !off )
		return ;
	char *d = cx.P<char>( off ) ;
	for ( int i = 0 ; i < n ; ++i )
		d[i] = s[i] ;
	d[n] = '\0' ;
	c->nameOff = off ;
	c->nameLen = n ;
}

// SeqSet::SetPrevAddInfo (SeqSet.hpp:627)
T4_D inline void t4_set_prev( T4Stream *st, int seqIdx, int readStart, int readEnd, int seqStart, int strand )
{
	st->prevSeqIdx = seqIdx ;
	st->prevReadStart = readStart ;
	st->prevReadEnd = readEnd ;
	st->prevSeqStart = seqStart ;
	st->prevStrand = strand ;
}

// SeqSet::ReverseComplement (SeqSet.hpp:2616)
T4_D inline void t4_revcomp( char *rc, const char *s, int len )
{
	for ( int i = 0 ; i < len ; ++i )
	{
		char c = s[len - 1 - i] ;
		rc[i] = ( c != 'N' ) ? t4_numToNuc( 3 - t4_nuc( c ) ) : 'N' ;
	}
	rc[len] = '\0' ;
}

// ---------------------------------------------------------------------------
// collective primitives
// ---------------------------------------------------------------------------
// Grow the hit scratch buffers to hold n keys.
T4_D inline void c_ensure_hits( T4Ctx &cx, u32 n )
{
	T4Stream *st = cx.st ;
	// the grow decision must be CTA-uniform (a barrier sits inside the branch): every thread reads the cap between
	// two barriers, before thread 0 can overwrite it
	T4_SYNC() ;
	const u32 capNow = st->hitCap ;
	T4_SYNC() ;
	if ( n + 1 > capNow )
	{
		if ( cx.tid == 0 )
		{
			u32 nc = capNow ;
			while ( nc < n + 1 )
				nc *= 2 ;
			u64 a = s_alloc( cx, (u64)nc * 8 ) ;
			u64 b = s_alloc( cx, (u64)nc * 8 ) ;
			u64 g = s_alloc( cx, (u64)( nc + 1 ) * 4 ) ;
			u64 r = s_alloc( cx, (u64)( nc + 1 ) * 4 ) ;
			if ( a && b && g && r )
			{
				st->keysAOff = a ; st->keysBOff = b ; st->grpOff = g ; st->runOff = r ;
				st->hitCap = nc ;
			}
		}
		T4_SYNC() ;
	}
}

T4_D inline void c_ensure_ovl( T4Ctx &cx, u32 n )
{
	T4Stream *st = cx.st ;
	T4_SYNC() ; // CTA-uniform decision, see c_ensure_hits
	const u32 capNow = st->ovlCap ;
	T4_SYNC() ;
	if ( n + 1 > capNow )
	{
		if ( cx.tid == 0 )
		{
			u32 nc = capNow ;
			while ( nc < n + 1 )
				nc *= 2 ;
			u64 a = s_alloc( cx, (u64)nc * sizeof( T4Ovl ) ) ;
			u64 b = s_alloc( cx, (u64)nc * sizeof( T4Ovl ) ) ;
			u64 c = s_alloc( cx, (u64)nc * sizeof( T4Ovl ) ) ;
			u64 d = s_alloc( cx, (u64)nc * sizeof( T4Ovl ) ) ;
			u64 e = s_alloc( cx, (u64)nc * 8 ) ;
			u64 f = s_alloc( cx, (u64)nc * 32 * 4 ) ;
			if ( a && b && c && d && e && f )
			{
				// the live overlaps (if any) stay valid: callers only grow before filling
				st->ovlOff = a ; st->ovlTmpOff = b ; st->extOff = c ; st->failOff = d ; st->anchorOff = e ; st->bitsOff = f ;
				st->ovlCap = nc ;
			}
		}
		T4_SYNC() ;
	}
}

// Exclusive scan of one value per thread; returns this thread's offset and the total.
T4_D inline u32 c_scan_threads( T4Ctx &cx, u32 v, u32 &total )
{
#if T4_CUDA
	// warp shuffle scan + one shared-memory hop across warps (blockDim is a multiple of 32)
	const int lane = cx.tid & 31, warp = cx.tid >> 5, nwarps = cx.nt >> 5 ;
	u32 inc = v ;
#pragma unroll
	for ( int d = 1 ; d < 32 ; d <<= 1 )
	{
		u32 t = __shfl_up_sync( 0xffffffffu, inc, d ) ;
		if ( lane >= d )
			inc += t ;
	}
	T4_SYNC() ; // previous users of sm->scan are done
	if ( lane == 31 )
		cx.sm->scan[warp] = inc ;
	T4_SYNC() ;
	u32 base = 0, tot = 0 ;
	for ( int w = 0 ; w < nwarps ; ++w )
	{
		u32 x = cx.sm->scan[w] ;
		if ( w < warp )
			base += x ;
		tot += x ;
	}
	total = tot ;
	return base + inc - v ;
#else
	T4_SYNC() ;
	cx.sm->scan[cx.tid] = v ;
	T4_SYNC() ;
	if ( cx.tid == 0 )
	{
		u32 s = 0 ;
		for ( int t = 0 ; t < cx.nt ; ++t )
		{
			u32 x = cx.sm->scan[t] ;
			cx.sm->scan[t] = s ;
			s += x ;
		}
		cx.sm->scan[cx.nt] = s ;
	}
	T4_SYNC() ;
	total = cx.sm->scan[cx.nt] ;
	return cx.sm->scan[cx.tid] ;
#endif
}

// Sort n keys ascending.  Returns the buffer (a or b) holding the result.
T4_D inline u64 *c_sort_keys( T4Ctx &cx, u64 *a, u64 *b, u32 n )
{
#if !T4_CUDA
	std::sort( a, a + n ) ;
	return a ;
#else
	if ( n <= 1 )
		return a ;
	if ( n <= T4_SMEM_SORT )
	{
		// small inputs (the common case for sharded streams): bitonic sort entirely in shared memory
		u64 *sk = (u64 *)cx.sm->radix ; // the radix counter area doubles as the sort buffer (u64[1024])
		u32 np = 1 ;
		while ( np < n )
			np <<= 1 ;
		for ( u32 i = cx.tid ; i < np ; i += cx.nt )
			sk[i] = i < n ? a[i] : ~0ull ;
		T4_SYNC() ;
		for ( u32 size = 2 ; size <= np ; size <<= 1 )
			for ( u32 stride = size >> 1 ; stride > 0 ; stride >>= 1 )
			{
				for ( u32 t = cx.tid ; t < np / 2 ; t += cx.nt )
				{
					u32 lo = 2 * t - ( t & ( stride - 1 ) ) ;
					u32 hi = lo + stride ;
					bool up = ( ( lo & size ) == 0 ) ;
					u64 x = sk[lo], y = sk[hi] ;
					if ( ( x > y ) == up )
					{
						sk[lo] = y ;
						sk[hi] = x ;
					}
				}
				T4_SYNC() ;
			}
		for ( u32 i = cx.tid ; i < n ; i += cx.nt )
			a[i] = sk[i] ;
		T4_SYNC() ;
		return a ;
	}
	// which bits vary at all?
	u64 vo = 0, va = ~0ull ;
	for ( u32 i = cx.tid ; i < n ; i += cx.nt )
	{
		u64 k = a[i] ;
		vo |= k ;
		va &= k ;
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
	{
		cx.sm->red[0] = 0 ;
		cx.sm->red[1] = ~0ull ;
	}
	T4_SYNC() ;
	atomicOr( (unsigned long long *)&cx.sm->red[0], (unsigned long long)vo ) ;
	atomicAnd( (unsigned long long *)&cx.sm->red[1], (unsigned long long)va ) ;
	T4_SYNC() ;
	u64 vary = cx.sm->red[0] ^ cx.sm->red[1] ;
	// LSD radix sort, 8-bit digits, one contiguous chunk of keys per WARP.  Within a warp keys are taken 32 at a time
	// in order; lanes with equal digits find each other with __match_any_sync and rank themselves by lane, so the
	// scatter is stable.  Counters: digit-major, warp-minor (256 x nwarps) in the shared radix area.
	const int lane = cx.tid & 31, warp = cx.tid >> 5, nwarps = cx.nt >> 5 ;
	const u32 wchunk = ( ( n + nwarps - 1 ) / nwarps + 31 ) & ~31u ;
	const u32 wlo = warp * wchunk < n ? warp * wchunk : n ;
	const u32 whi = wlo + wchunk < n ? wlo + wchunk : n ;
	const unsigned lt = ( 1u << lane ) - 1u ;
	u32 *cnt = cx.sm->radix ; // [256][nwarps]
	u64 *src = a, *dst = b ;
	for ( int shift = 0 ; shift < 64 ; shift += 8 )
	{
		if ( ( ( vary >> shift ) & 255 ) == 0 )
			continue ;
		for ( int x = cx.tid ; x < 256 * nwarps ; x += cx.nt )
			cnt[x] = 0 ;
		T4_SYNC() ;
		for ( u32 i0 = wlo ; i0 < whi ; i0 += 32 )
		{
			u32 i = i0 + lane ;
			bool have = i < whi ;
			u32 d = have ? (u32)( ( src[i] >> shift ) & 255 ) : 256u + lane ; // idle lanes get private pseudo digits
			unsigned peers = __match_any_sync( 0xffffffffu, d ) ;
			if ( have && ( peers & lt ) == 0 )
				cnt[d * nwarps + warp] += __popc( peers ) ;
			__syncwarp() ;
		}
		T4_SYNC() ;
		// exclusive scan of the 256 * nwarps counters (digit major): each thread takes a contiguous piece
		{
			const int total = 256 * nwarps ;
			const int per = ( total + cx.nt - 1 ) / cx.nt ;
			const int lo2 = cx.tid * per < total ? cx.tid * per : total ;
			const int hi2 = lo2 + per < total ? lo2 + per : total ;
			u32 sum = 0 ;
			for ( int x = lo2 ; x < hi2 ; ++x )
				sum += cnt[x] ;
			u32 tot ;
			u32 base = c_scan_threads( cx, sum, tot ) ;
			for ( int x = lo2 ; x < hi2 ; ++x )
			{
				u32 v = cnt[x] ;
				cnt[x] = base ;
				base += v ;
			}
		}
		T4_SYNC() ;
		for ( u32 i0 = wlo ; i0 < whi ; i0 += 32 )
		{
			u32 i = i0 + lane ;
			bool have = i < whi ;
			u64 k = have ? src[i] : 0 ;
			u32 d = have ? (u32)( ( k >> shift ) & 255 ) : 256u + lane ;
			unsigned peers = __match_any_sync( 0xffffffffu, d ) ;
			u32 pos = 0 ;
			if ( have )
				pos = cnt[d * nwarps + warp] + __popc( peers & lt ) ;
			__syncwarp() ;
			if ( have )
			{
				dst[pos] = k ;
				if ( ( peers & lt ) == 0 )
					cnt[d * nwarps + warp] += __popc( peers ) ;
			}
			__syncwarp() ;
		}
		T4_SYNC() ;
		u64 *t = src ; src = dst ; dst = t ;
	}
	return src ;
#endif
}

// ---------------------------------------------------------------------------
// the main hit sort of GetOverlapsFromRead: a stable sort on the key prefix (strand | contig | diagonal)
// ---------------------------------------------------------------------------
// Up to T4_HIT_TILE keys are sorted and chained in dynamic shared memory (two buffers of T4_HIT_TILE + 1 keys; the
// stream and aux kernels are launched with T4_HIT_TILE_BYTES of it), more in global memory.  No tile size costs
// occupancy (the kernels stay register bound at 4 CTAs per SM), but the tile comes out of L1, through which the other
// phases read contigs, postings and posWeight.  One default bench.py workload on an H100 80GB HBM3 (700 W), ms per
// step against 583 for the parent's sort: a 2048-key tile 602, 1024 keys 565, 512 keys 556, no tile 556.
#ifndef T4_HIT_TILE
#define T4_HIT_TILE 512
#endif
#define T4_HIT_TILE_BYTES ( 2 * ( T4_HIT_TILE + 1 ) * 8 )
#define T4_PREFIX_DIGIT 9 // widest radix digit: 2^9 counters per warp fill the radix area at 4 warps
static_assert( T4_HIT_TILE <= T4_RADIX * T4_MAX_NT, "a run's hit length per run lives in the radix area" ) ;
static_assert( ( 1 << T4_PREFIX_DIGIT ) * ( T4_MAX_NT / 32 ) <= T4_RADIX * T4_MAX_NT, "radix counters" ) ;
#if T4_CUDA
extern __shared__ __align__( 16 ) u64 t4_hit_tile[] ;
#endif

// The sorted hits as the chain pass reads them: keys (shared or global memory) and room for the group and run heads
// (H + 1 each) and a hit length per run (H).
struct T4HitView
{
	const u64 *keys ;
	u32 *grp, *run, *hl ;
} ;

// Exclusive scans of two values per thread at once.
T4_D inline void c_scan_threads2( T4Ctx &cx, u32 v0, u32 v1, u32 &o0, u32 &o1, u32 &t0, u32 &t1 )
{
#if T4_CUDA
	const int lane = cx.tid & 31, warp = cx.tid >> 5, nwarps = cx.nt >> 5 ;
	u32 i0 = v0, i1 = v1 ;
#pragma unroll
	for ( int d = 1 ; d < 32 ; d <<= 1 )
	{
		u32 x0 = __shfl_up_sync( 0xffffffffu, i0, d ) ;
		u32 x1 = __shfl_up_sync( 0xffffffffu, i1, d ) ;
		if ( lane >= d )
		{
			i0 += x0 ;
			i1 += x1 ;
		}
	}
	T4_SYNC() ;
	if ( lane == 31 )
	{
		cx.sm->scan[warp] = i0 ;
		cx.sm->scan[T4_MAX_NT / 32 + warp] = i1 ;
	}
	T4_SYNC() ;
	u32 b0 = 0, b1 = 0, s0 = 0, s1 = 0 ;
	for ( int w = 0 ; w < nwarps ; ++w )
	{
		u32 x0 = cx.sm->scan[w], x1 = cx.sm->scan[T4_MAX_NT / 32 + w] ;
		if ( w < warp )
		{
			b0 += x0 ;
			b1 += x1 ;
		}
		s0 += x0 ;
		s1 += x1 ;
	}
	o0 = b0 + i0 - v0 ;
	o1 = b1 + i1 - v1 ;
	t0 = s0 ;
	t1 = s1 ;
#else
	o0 = c_scan_threads( cx, v0, t0 ) ;
	o1 = c_scan_threads( cx, v1, t1 ) ;
#endif
}

// One neighbour-compare pass over the sorted keys: group heads (strand or contig changes) and run heads (the diagonal
// changes too) in order, grp[nG] = run[nR] = n.  Every group head is a run head.
T4_D inline void c_hit_heads( T4Ctx &cx, const u64 *keys, u32 n, u32 *grp, u32 *run, u32 &nG, u32 &nR )
{
	u32 chunk = ( n + cx.nt - 1 ) / cx.nt ;
	u32 lo = cx.tid * chunk ;
	u32 hi = lo + chunk < n ? lo + chunk : n ;
	if ( lo > n )
		lo = n ;
	u32 cg = 0, cr = 0 ;
	u64 prev = lo > 0 && lo < hi ? keys[lo - 1] : 0 ;
	for ( u32 i = lo ; i < hi ; ++i )
	{
		u64 k = keys[i] ;
		cg += i == 0 || ( k >> T4_KEY_IDX_SHIFT ) != ( prev >> T4_KEY_IDX_SHIFT ) ;
		cr += i == 0 || ( k >> T4_KEY_C_SHIFT ) != ( prev >> T4_KEY_C_SHIFT ) ;
		prev = k ;
	}
	u32 og, orr ;
	c_scan_threads2( cx, cg, cr, og, orr, nG, nR ) ;
	prev = lo > 0 && lo < hi ? keys[lo - 1] : 0 ;
	for ( u32 i = lo ; i < hi ; ++i )
	{
		u64 k = keys[i] ;
		if ( i == 0 || ( k >> T4_KEY_IDX_SHIFT ) != ( prev >> T4_KEY_IDX_SHIFT ) )
			grp[og++] = i ;
		if ( i == 0 || ( k >> T4_KEY_C_SHIFT ) != ( prev >> T4_KEY_C_SHIFT ) )
			run[orr++] = i ;
		prev = k ;
	}
	if ( cx.tid == 0 )
	{
		grp[nG] = n ;
		run[nR] = n ;
	}
	T4_SYNC() ;
}

#if T4_CUDA
// Order-preserving map of a key's prefix onto few bits: (strand, contig - min contig, diagonal - min diagonal), each
// field only as wide as its range over the read; invalid keys map above every valid one.
struct T4PrefixRank
{
	u32 idxMin, cMin ;
	int cb, sShift, tb ;

	T4_D u64 operator()( u64 k ) const
	{
		if ( k == T4_KEY_INVALID )
			return 1ull << tb ;
		u64 r = ( (u64)( (u32)t4_key_idx( k ) - idxMin ) << cb ) | (u64)( (u32)( ( k >> T4_KEY_C_SHIFT ) & T4_KEY_C_MASK ) - cMin ) ;
		if ( sShift >= 0 )
			r |= ( k >> T4_KEY_STRAND_SHIFT ) << sShift ;
		return r ;
	}
} ;

T4_D inline int t4_bits( u32 x ) { return x ? 32 - __clz( x ) : 0 ; }
#endif

// Sorts the n keys of a[] (in c_get_hits' emission order) ascending and returns the global buffer holding them, a or
// b, for scoring; *v says where the chain pass reads them and where it keeps its heads.
//
// The device sorts on the prefix key >> T4_KEY_C_SHIFT only, stably, and that gives the order of a sort on the whole
// key: c_get_hits emits its hits in ascending (pass, q) order (the prefix sum and the serial walk both reserve slots
// in q order, and a long list is copied into its own reserved slots), so within one (strand, contig, diagonal) the
// hits come in ascending q, and b = q - c ascends with q.  Two hits never share (strand, contig, diagonal, b): the
// diagonal and b fix q, and one position's postings are distinct (contig, offset) pairs, so the repeat flag (bit 0)
// never breaks a tie.  Invalid keys (~0) sort last.  This does not hold for the other sorts (SortHits order, the
// reference sets): they keep c_sort_keys.
T4_D inline u64 *c_sort_hit_prefix( T4Ctx &cx, u64 *a, u64 *b, u32 n, T4HitView *v )
{
	T4Stream *st = cx.st ;
#if !T4_CUDA
	std::sort( a, a + n ) ;
	v->keys = a ;
	v->grp = cx.P<u32>( st->grpOff ) ;
	v->run = cx.P<u32>( st->runOff ) ;
	v->hl = (u32 *)b ;
	return a ;
#else
	const bool tile = n <= T4_HIT_TILE ;
	u64 *src = tile ? t4_hit_tile : a, *dst = tile ? t4_hit_tile + T4_HIT_TILE + 1 : b ;
	{
		// the ranges of the prefix fields; the tile is filled on the way
		u32 iMin = ~0u, iMax = 0, cMin = ~0u, cMax = 0, sOr = 0, sAnd = 1, inv = 0 ;
		for ( u32 i = cx.tid ; i < n ; i += cx.nt )
		{
			u64 k = a[i] ;
			if ( tile )
				src[i] = k ;
			if ( k == T4_KEY_INVALID )
			{
				inv = 1 ;
				continue ;
			}
			u32 ix = (u32)t4_key_idx( k ), c = (u32)( ( k >> T4_KEY_C_SHIFT ) & T4_KEY_C_MASK ), s = (u32)( k >> T4_KEY_STRAND_SHIFT ) ;
			iMin = min( iMin, ix ) ;
			iMax = max( iMax, ix ) ;
			cMin = min( cMin, c ) ;
			cMax = max( cMax, c ) ;
			sOr |= s ;
			sAnd &= s ;
		}
		const int lane = cx.tid & 31, warp = cx.tid >> 5, nwarps = cx.nt >> 5 ;
		iMin = __reduce_min_sync( 0xffffffffu, iMin ) ;
		iMax = __reduce_max_sync( 0xffffffffu, iMax ) ;
		cMin = __reduce_min_sync( 0xffffffffu, cMin ) ;
		cMax = __reduce_max_sync( 0xffffffffu, cMax ) ;
		sOr = __reduce_or_sync( 0xffffffffu, sOr ) ;
		sAnd = __reduce_and_sync( 0xffffffffu, sAnd ) ;
		inv = __reduce_or_sync( 0xffffffffu, inv ) ;
		T4_SYNC() ; // earlier readers of sm->scan are done
		if ( lane == 0 )
		{
			u32 *w = cx.sm->scan + 7 * warp ;
			w[0] = iMin ; w[1] = iMax ; w[2] = cMin ; w[3] = cMax ; w[4] = sOr ; w[5] = sAnd ; w[6] = inv ;
		}
		T4_SYNC() ;
		for ( int x = 0 ; x < nwarps ; ++x )
		{
			const u32 *w = cx.sm->scan + 7 * x ;
			iMin = min( iMin, w[0] ) ; iMax = max( iMax, w[1] ) ; cMin = min( cMin, w[2] ) ; cMax = max( cMax, w[3] ) ;
			sOr |= w[4] ; sAnd &= w[5] ; inv |= w[6] ;
		}
		const bool anyValid = iMin <= iMax ;
		T4PrefixRank rank ;
		rank.idxMin = iMin ;
		rank.cMin = cMin ;
		rank.cb = anyValid ? t4_bits( cMax - cMin ) : 0 ;
		const int ib = anyValid ? t4_bits( iMax - iMin ) : 0 ;
		const int sb = ( anyValid && sOr != sAnd ) ? 1 : 0 ;
		rank.sShift = sb ? rank.cb + ib : -1 ;
		rank.tb = rank.cb + ib + sb ;
		const int nb = rank.tb + (int)inv ;
		// LSD radix over the rank in digits of equal width (at most T4_PREFIX_DIGIT bits), one contiguous chunk of keys
		// per warp; lanes with equal digits find each other with __match_any_sync and rank themselves by lane, so the
		// scatter is stable.  Counters: digit-major, warp-minor, in the radix area.
		const int passes = ( nb + T4_PREFIX_DIGIT - 1 ) / T4_PREFIX_DIGIT ;
		const int width = passes ? ( nb + passes - 1 ) / passes : 0 ;
		const u32 D = 1u << width ;
		const u32 wchunk = ( ( n + nwarps - 1 ) / nwarps + 31 ) & ~31u ;
		const u32 wlo = warp * wchunk < n ? warp * wchunk : n ;
		const u32 whi = wlo + wchunk < n ? wlo + wchunk : n ;
		const unsigned lt = ( 1u << lane ) - 1u ;
		u32 *cnt = cx.sm->radix ;
		for ( int shift = 0 ; shift < nb ; shift += width )
		{
			for ( u32 x = cx.tid ; x < D * nwarps ; x += cx.nt )
				cnt[x] = 0 ;
			T4_SYNC() ;
			for ( u32 i0 = wlo ; i0 < whi ; i0 += 32 )
			{
				u32 i = i0 + lane ;
				bool have = i < whi ;
				u32 d = have ? (u32)( rank( src[i] ) >> shift ) & ( D - 1 ) : D + lane ; // idle lanes: private pseudo digits
				unsigned peers = __match_any_sync( 0xffffffffu, d ) ;
				if ( have && ( peers & lt ) == 0 )
					cnt[d * nwarps + warp] += __popc( peers ) ;
				__syncwarp() ;
			}
			T4_SYNC() ;
			{
				const int total = (int)D * nwarps ;
				const int per = ( total + cx.nt - 1 ) / cx.nt ;
				const int lo2 = cx.tid * per < total ? cx.tid * per : total ;
				const int hi2 = lo2 + per < total ? lo2 + per : total ;
				u32 sum = 0 ;
				for ( int x = lo2 ; x < hi2 ; ++x )
					sum += cnt[x] ;
				u32 tot ;
				u32 base = c_scan_threads( cx, sum, tot ) ;
				for ( int x = lo2 ; x < hi2 ; ++x )
				{
					u32 c = cnt[x] ;
					cnt[x] = base ;
					base += c ;
				}
			}
			T4_SYNC() ;
			for ( u32 i0 = wlo ; i0 < whi ; i0 += 32 )
			{
				u32 i = i0 + lane ;
				bool have = i < whi ;
				u64 k = have ? src[i] : 0 ;
				u32 d = have ? (u32)( rank( k ) >> shift ) & ( D - 1 ) : D + lane ;
				unsigned peers = __match_any_sync( 0xffffffffu, d ) ;
				u32 pos = 0 ;
				if ( have )
					pos = cnt[d * nwarps + warp] + __popc( peers & lt ) ;
				__syncwarp() ;
				if ( have )
				{
					dst[pos] = k ;
					if ( ( peers & lt ) == 0 )
						cnt[d * nwarps + warp] += __popc( peers ) ;
				}
				__syncwarp() ;
			}
			T4_SYNC() ;
			u64 *t = src ; src = dst ; dst = t ;
		}
	}
	v->keys = src ;
	if ( !tile )
	{
		v->grp = cx.P<u32>( st->grpOff ) ;
		v->run = cx.P<u32>( st->runOff ) ;
		v->hl = (u32 *)dst ;
		return src ;
	}
	// scoring reads the keys after the tile is gone: one coalesced copy out.  The other buffer holds the heads
	// (2 n + 2 <= 2 T4_HIT_TILE + 2 words), the radix area the hit lengths.
	for ( u32 i = cx.tid ; i < n ; i += cx.nt )
		a[i] = src[i] ;
	v->run = (u32 *)dst ;
	v->grp = (u32 *)dst + n + 1 ;
	v->hl = cx.sm->radix ;
	return a ;
#endif
}

// ---------------------------------------------------------------------------
// banded global alignment against posWeight columns
// ---------------------------------------------------------------------------
// AlignAlgo::IsBaseEqual (AlignAlgo.hpp:49-55)
T4_HD inline bool t4_base_equal( const int *w, char c )
{
	int sum = w[0] + w[1] + w[2] + w[3] ;
	if ( sum == 0 || c == 'N' || sum < 3 * w[t4_nuc( c )] )
		return true ;
	return false ;
}

// AlignAlgo::GlobalAlignment_PosWeight (AlignAlgo.hpp:57-216).  tw: lent columns of int[4]; p: lenp chars.
// rows: 2*W ints, act: (lenp+1)*W bytes with W = leftBand + rightBand + 3.  Scores are kept for two rows only;
// the traceback decision of every band cell (a pure function of the cell and its three neighbours,
// AlignAlgo.hpp:177-193) is taken while filling and stored as one byte.
T4_HD inline int t4_dp_posweight( const int *tw, int lent, const char *p, int lenp, signed char *align, int *rows,
	unsigned char *act, int *usedFullDp )
{
	if ( usedFullDp )
		*usedFullDp = 0 ;
	if ( lent == 0 || lenp == 0 )
	{
		align[0] = -1 ;
		return 0 ;
	}
	else if ( lent == 1 && lenp == 1 )
	{
		if ( t4_base_equal( tw, p[0] ) )
		{
			align[0] = EDIT_MATCH ;
			align[1] = -1 ;
			return SCORE_MATCH ;
		}
		align[0] = EDIT_MISMATCH ;
		align[1] = -1 ;
		return SCORE_MISMATCH ;
	}
	int i, j ;
	if ( lent == lenp )
	{
		int score = 0 ;
		for ( i = 0 ; i < lent ; ++i )
		{
			if ( t4_base_equal( tw + 4 * i, p[i] ) )
			{
				align[i] = EDIT_MATCH ;
				score += SCORE_MATCH ;
			}
			else
			{
				align[i] = EDIT_MISMATCH ;
				score += SCORE_MISMATCH ;
			}
		}
		align[i] = -1 ;
		if ( score >= lent * SCORE_MATCH + 2 * SCORE_INDEL )
			return score ;
	}
	if ( usedFullDp )
		*usedFullDp = 1 ;
	int leftBand = T4_DP_BAND, rightBand = T4_DP_BAND ;
	if ( lent > lenp )
		rightBand += lent - lenp ;
	else if ( lent < lenp )
		leftBand += lenp - lent ;
	const int W = leftBand + rightBand + 3 ;
	const int negInf = ( lent + 1 ) * ( lenp + 1 ) * SCORE_INDEL ;
	int *prev = rows, *cur = rows + W ;
	// row 0: m[0][j] = j ? -4 - 4j : 0 (AlignAlgo.hpp:120-129)
	{
		int wlo = 0 - leftBand - 1 ;
		for ( int l = 0 ; l < W ; ++l )
		{
			j = wlo + l ;
			prev[l] = ( j == 0 ) ? 0 : ( SCORE_INDEL + j * SCORE_INDEL ) ;
		}
	}
	for ( i = 1 ; i <= lenp ; ++i )
	{
		int wlo = i - leftBand - 1 ;
		int start = ( i - leftBand < 1 ) ? 1 : ( i - leftBand ) ;
		int end = ( i + rightBand > lent ) ? lent : ( i + rightBand ) ;
		if ( 0 >= wlo )
			cur[0 - wlo] = SCORE_INDEL + i * SCORE_INDEL ;
		if ( start > 1 )
			cur[start - 1 - wlo] = negInf ;
		if ( end < lent )
			cur[end + 1 - wlo] = negInf ;
		unsigned char *arow = act + (size_t)i * W ;
		char pc = p[i - 1] ;
		for ( j = start ; j <= end ; ++j )
		{
			int l = j - wlo ;
			int diff = t4_base_equal( tw + 4 * ( j - 1 ), pc ) ? SCORE_MATCH : SCORE_MISMATCH ;
			int dg = prev[l] + diff ;          // (i-1, j-1)
			int lf = cur[l - 1] + SCORE_INDEL ; // (i, j-1)
			int up = prev[l + 1] + SCORE_INDEL ; // (i-1, j)
			int score = dg ;
			if ( lf > score ) score = lf ;
			if ( up > score ) score = up ;
			cur[l] = score ;
			int a = 0 ;
			if ( lf == score ) a = EDIT_DELETE ;
			if ( up == score ) a = EDIT_INSERT ;
			if ( dg == score ) a = ( diff == SCORE_MATCH ) ? EDIT_MATCH : EDIT_MISMATCH ;
			arow[l] = (unsigned char)a ;
		}
		int *t = prev ; prev = cur ; cur = t ;
	}
	int ret = prev[lent - ( lenp - leftBand - 1 )] ;
	// trace back (AlignAlgo.hpp:168-214)
	int tagi = lenp, tagj = lent, tag = 0 ;
	while ( tagi > 0 || tagj > 0 )
	{
		int a ;
		if ( tagi > 0 && tagj > 0 )
			a = act[(size_t)tagi * W + ( tagj - ( tagi - leftBand - 1 ) )] ;
		else if ( tagj > 0 ) // row 0: m[0][j-1] - 4 == m[0][j] holds iff j >= 2
			a = ( tagj >= 2 ) ? EDIT_DELETE : EDIT_MATCH ;
		else // column 0
			a = ( tagi >= 2 ) ? EDIT_INSERT : EDIT_MATCH ;
		align[tag] = (signed char)a ;
		++tag ;
		if ( a == EDIT_DELETE )
			--tagj ;
		else if ( a == EDIT_INSERT )
			--tagi ;
		else
		{
			--tagi ;
			--tagj ;
		}
	}
	align[tag] = -1 ;
	for ( i = 0, j = tag - 1 ; i < j ; ++i, --j )
	{
		signed char tmp = align[i] ;
		align[i] = align[j] ;
		align[j] = tmp ;
	}
	return ret ;
}

// n independent GlobalAlignment_PosWeight problems (t4_dp_kernel): problem i aligns p[pOff[i] .. pOff[i + 1]) to the
// columns tw[4 tOff[i] .. 4 tOff[i + 1]) into align + alignOff[i], with its rows and traceback at scratch + scratchOff[i].
struct T4DpParams
{
	const int *tw ;
	const i64 *tOff ;
	const char *p ;
	const i64 *pOff ;
	signed char *align ;
	const i64 *alignOff ;
	int *score ;
	char *scratch ;
	const i64 *scratchOff ;
	int n ;
} ;

T4_HD inline void t4_dp_one( const T4DpParams &P, i64 i )
{
	int lent = (int)( P.tOff[i + 1] - P.tOff[i] ) ;
	int lenp = (int)( P.pOff[i + 1] - P.pOff[i] ) ;
	int d = lent > lenp ? lent - lenp : lenp - lent ;
	int W = 2 * T4_DP_BAND + 3 + d ;
	char *s = P.scratch + P.scratchOff[i] ;
	P.score[i] = t4_dp_posweight( P.tw + 4 * P.tOff[i], lent, P.p + P.pOff[i], lenp, P.align + P.alignOff[i], (int *)s,
		(unsigned char *)( s + 8 * W ), 0 ) ;
}

// The same alignment for lent == lenp == n (every hot-path call: overhangs and same-diagonal gaps), band +-5.
// Both score rows live in registers (the 13-wide window is fully unrolled), IsBaseEqual outcomes slide through a
// 64-bit register as one nibble per column (bit b = "base b equals this column"), and the traceback decision of a
// row is packed into one 32-bit word (2 bits per band cell).  act32: n + 1 words.
T4_HD inline int t4_dp_equal( const int *tw, const char *p, int n, signed char *align, u32 *act32, bool diagKnownBad, int *usedFullDp )
{
	if ( usedFullDp )
		*usedFullDp = 0 ;
	if ( n == 0 )
	{
		align[0] = -1 ;
		return 0 ;
	}
	if ( n == 1 )
	{
		bool eq = t4_base_equal( tw, p[0] ) ;
		align[0] = eq ? EDIT_MATCH : EDIT_MISMATCH ;
		align[1] = -1 ;
		return eq ? SCORE_MATCH : SCORE_MISMATCH ;
	}
	if ( !diagKnownBad )
	{
		int score = 0 ;
		for ( int i = 0 ; i < n ; ++i )
		{
			if ( t4_base_equal( tw + 4 * i, p[i] ) )
			{
				align[i] = EDIT_MATCH ;
				score += SCORE_MATCH ;
			}
			else
			{
				align[i] = EDIT_MISMATCH ;
				score += SCORE_MISMATCH ;
			}
		}
		align[n] = -1 ;
		if ( score >= n * SCORE_MATCH + 2 * SCORE_INDEL )
			return score ;
	}
	if ( usedFullDp )
		*usedFullDp = 1 ;
	const int negInf = ( n + 1 ) * ( n + 1 ) * SCORE_INDEL ;
	int prev[13], cur[13] ;
	// row 0, window columns j = l - 6
#pragma unroll
	for ( int l = 0 ; l < 13 ; ++l )
	{
		int j = l - 6 ;
		prev[l] = ( j == 0 ) ? 0 : ( SCORE_INDEL + j * SCORE_INDEL ) ;
	}
	// eq nibble of window slot l (column j = wlo + l, posWeight index j - 1) at bits [4l, 4l+4)
	unsigned long long eqw = 0 ;
#pragma unroll
	for ( int l = 1 ; l <= 11 ; ++l )
	{
		int c = l - 6 ; // posWeight index for row 1: j - 1 with j = (1 - 6) + l
		if ( c >= 0 && c < n )
			eqw |= (unsigned long long)t4_eq_nibble( tw + 4 * c ) << ( 4 * l ) ;
	}
	for ( int i = 1 ; i <= n ; ++i )
	{
		const int wlo = i - 6 ;
		const int start = ( i - 5 < 1 ) ? 1 : ( i - 5 ) ;
		const int end = ( i + 5 > n ) ? n : ( i + 5 ) ;
		const char pc = p[i - 1] ;
		const int pn = t4_nuc( pc ) ;
		const bool pN = ( pc == 'N' ) ;
		u32 arow = 0 ;
		if ( i >= 7 && i + 5 <= n )
		{
			// interior row: the whole 11-cell band is inside the matrix, both window edges are -inf
			const unsigned long long rowEq = pN ? ~0ull : ( eqw >> pn ) ;
			cur[0] = negInf ;
			cur[12] = negInf ;
#pragma unroll
			for ( int l = 1 ; l <= 11 ; ++l )
			{
				bool eq = ( (unsigned)( rowEq >> ( 4 * l ) ) & 1u ) != 0 ;
				int dg = prev[l] + ( eq ? SCORE_MATCH : SCORE_MISMATCH ) ;
				int lf = cur[l - 1] + SCORE_INDEL ;
				int up = prev[l + 1] + SCORE_INDEL ;
				int score = dg ;
				if ( lf > score ) score = lf ;
				if ( up > score ) score = up ;
				cur[l] = score ;
				u32 a = ( dg == score ) ? ( eq ? (u32)EDIT_MATCH : (u32)EDIT_MISMATCH ) : ( ( up == score ) ? (u32)EDIT_INSERT : (u32)EDIT_DELETE ) ;
				arow |= a << ( 2 * l ) ;
			}
		}
		else
		{
	#pragma unroll
			for ( int l = 0 ; l < 13 ; ++l )
				cur[l] = negInf ;
			if ( wlo <= 0 )
			{
				// column 0 sits at slot -wlo (0..5)
	#pragma unroll
				for ( int l = 0 ; l <= 5 ; ++l )
					if ( l == -wlo )
						cur[l] = SCORE_INDEL + i * SCORE_INDEL ;
			}
	#pragma unroll
			for ( int l = 1 ; l <= 11 ; ++l )
			{
				int j = wlo + l ;
				if ( j >= start && j <= end )
				{
					bool eq = pN || ( ( (unsigned)( eqw >> ( 4 * l ) ) >> pn ) & 1u ) ;
					int diff = eq ? SCORE_MATCH : SCORE_MISMATCH ;
					int dg = prev[l] + diff ;
					int lf = cur[l - 1] + SCORE_INDEL ;
					int up = prev[l + 1] + SCORE_INDEL ;
					int score = dg ;
					if ( lf > score ) score = lf ;
					if ( up > score ) score = up ;
					cur[l] = score ;
					u32 a = 0 ;
					if ( lf == score ) a = EDIT_DELETE ;
					if ( up == score ) a = EDIT_INSERT ;
					if ( dg == score ) a = eq ? EDIT_MATCH : EDIT_MISMATCH ;
					arow |= a << ( 2 * l ) ;
				}
			}
		}
		act32[i] = arow ;
#pragma unroll
		for ( int l = 0 ; l < 13 ; ++l )
			prev[l] = cur[l] ;
		// slide the eq window: slot l of row i+1 is slot l+1 of row i; new column at slot 11 has posWeight index i + 5
		eqw >>= 4 ;
		eqw &= ~( 0xFull << 44 ) ;
		if ( i + 5 < n )
			eqw |= (unsigned long long)t4_eq_nibble( tw + 4 * ( i + 5 ) ) << 44 ;
	}
	int ret = prev[6] ; // column n of row n: slot n - (n - 6)
	int tagi = n, tagj = n, tag = 0 ;
	while ( tagi > 0 || tagj > 0 )
	{
		int a ;
		if ( tagi > 0 && tagj > 0 )
			a = (int)( ( act32[tagi] >> ( 2 * ( tagj - ( tagi - 6 ) ) ) ) & 3u ) ;
		else if ( tagj > 0 )
			a = ( tagj >= 2 ) ? EDIT_DELETE : EDIT_MATCH ;
		else
			a = ( tagi >= 2 ) ? EDIT_INSERT : EDIT_MATCH ;
		align[tag] = (signed char)a ;
		++tag ;
		if ( a == EDIT_DELETE )
			--tagj ;
		else if ( a == EDIT_INSERT )
			--tagi ;
		else
		{
			--tagi ;
			--tagj ;
		}
	}
	align[tag] = -1 ;
	for ( int i = 0, j = tag - 1 ; i < j ; ++i, --j )
	{
		signed char tmp = align[i] ;
		align[i] = align[j] ;
		align[j] = tmp ;
	}
	return ret ;
}

// SeqSet::GetAlignStats (SeqSet.hpp:570)
T4_HD inline void t4_align_stats( const signed char *align, bool update, int &matchCnt, int &mismatchCnt, int &indelCnt )
{
	if ( !update )
		matchCnt = mismatchCnt = indelCnt = 0 ;
	for ( int k = 0 ; align[k] != -1 ; ++k )
	{
		if ( align[k] == EDIT_MATCH )
			++matchCnt ;
		else if ( align[k] == EDIT_MISMATCH )
			++mismatchCnt ;
		else
			++indelCnt ;
	}
}

struct T4DpScratch
{
	int *rows ;
	unsigned char *act ;
	signed char *align ;
} ;

T4_D inline T4DpScratch t4_dp_scratch( T4Ctx &cx )
{
	char *b = cx.P<char>( cx.st->dpOff ) + (size_t)cx.tid * cx.st->dpStride ;
	T4DpScratch s ;
	s.rows = (int *)b ;
	s.act = (unsigned char *)( b + 2 * T4_DP_W * 4 + 8 ) ;
	s.align = (signed char *)( b + 2 * T4_DP_W * 4 + 8 + ( T4_DEV_MAX_READ + 1 ) * T4_DP_W + 8 ) ;
	return s ;
}
T4_D inline T4DpScratch t4_dp_scratch_of( T4Ctx &cx, int tid )
{
	char *b = cx.P<char>( cx.st->dpOff ) + (size_t)tid * cx.st->dpStride ;
	T4DpScratch s ;
	s.rows = (int *)b ;
	s.act = (unsigned char *)( b + 2 * T4_DP_W * 4 + 8 ) ;
	s.align = (signed char *)( b + 2 * T4_DP_W * 4 + 8 + ( T4_DEV_MAX_READ + 1 ) * T4_DP_W + 8 ) ;
	return s ;
}
#define T4_DP_STRIDE ( ( 2 * T4_DP_W * 4 + 8 + ( T4_DEV_MAX_READ + 1 ) * T4_DP_W + 8 + 2 * T4_DEV_MAX_READ + 16 + 15 ) & ~15 )

// ---------------------------------------------------------------------------
// seeds: SeqSet::GetHitsFromRead (SeqSet.hpp:1341-1501), emitted as keys
// ---------------------------------------------------------------------------
// Reads cx.sm->read / rc.  Returns the number of keys written to keysA (invalid keys included,
// they sort last); *nValid receives the number of hits that survive the barcode filter.
// refSet: the set holds reference sequences (seqs[0].isRef): skipLimit = 0 (SeqSet.hpp:1351-1353), i.e. the >= 100 postings
// rule never skips; a compile-time `false` at the assembly path's call sites.
T4_D inline u32 c_get_hits( T4Ctx &cx, int len, int strand, int barcode, bool allowTotalSkip, int *anyBig, bool refSet = false )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	const int k = st->kmerLength ;
	T4Pos *pos = cx.P<T4Pos>( st->posOff ) ;
	const int m = len - k + 1 ; // positions per pass, index q = i - (k-1)
	// directory probes for every k-mer of both strand passes, in parallel.  Whether a probe "counts"
	// (SeqSet.hpp:1376: first k-mer, or code differs from prevKmerCode) is decided below, because the
	// reference's `continue` statements skip the prevKmerCode update.
	if ( cx.tid == 0 )
		sm->bi[2] = 0 ;
	T4_SYNC() ;
	for ( int x = cx.tid ; x < 2 * m ; x += cx.nt )
	{
		int pass = x >= m ;
		int q = pass ? x - m : x ;
		T4Pos *po = pos + pass * T4_DEV_MAX_READ + q ;
		po->cnt = 0 ;
		po->listOff = 0 ;
		po->base = 0xffffffffu ;
		if ( ( pass == 0 && strand == -1 ) || ( pass == 1 && strand == 1 ) )
			continue ;
		const char *r = pass ? sm->rc : sm->read ;
		u64 code = 0 ;
		bool valid = true ;
		for ( int j = 0 ; j < k ; ++j )
		{
			char c = r[q + j] ;
			code = ( code << 2 ) | (u64)t4_nuc( c ) ;
			if ( c == 'N' )
				valid = false ;
		}
		po->code = code ;
		if ( valid )
		{
			T4Dir *d = t4_dir_find( cx, t4_index_key( st, code, barcode ) ) ;
			if ( d )
			{
				po->cnt = d->cnt ;
				po->listOff = d->listOff ;
				if ( d->cnt >= 100 )
					sm->bi[2] = 1 ;
			}
		}
	}
	T4_SYNC() ;
	const bool anyLarge = sm->bi[2] != 0 ;
	T4_SYNC() ;
	if ( !anyLarge )
	{
		// no list reaches 100 postings: neither skip rule can fire, prevKmerCode is always the previous k-mer,
		// so "taken" is a per-position predicate and the hit slots are an exclusive prefix sum
		int tot = 2 * m ;
		int chunk = ( tot + cx.nt - 1 ) / cx.nt ;
		int lo = cx.tid * chunk ;
		int hi = lo + chunk < tot ? lo + chunk : tot ;
		u32 cnt = 0, looks = 0 ;
		for ( int x = lo ; x < hi ; ++x )
		{
			int pass = x >= m ;
			int q = pass ? x - m : x ;
			if ( ( pass == 0 && strand == -1 ) || ( pass == 1 && strand == 1 ) )
				continue ;
			T4Pos *po = pos + pass * T4_DEV_MAX_READ + q ;
			if ( q == 0 || po->code != po[-1].code )
			{
				++looks ;
				cnt += po->cnt ;
			}
		}
		u32 total ;
		u32 o = c_scan_threads( cx, cnt, total ) ;
		for ( int x = lo ; x < hi ; ++x )
		{
			int pass = x >= m ;
			int q = pass ? x - m : x ;
			if ( ( pass == 0 && strand == -1 ) || ( pass == 1 && strand == 1 ) )
				continue ;
			T4Pos *po = pos + pass * T4_DEV_MAX_READ + q ;
			if ( ( q == 0 || po->code != po[-1].code ) && po->cnt > 0 )
			{
				po->base = o ;
				o += po->cnt ;
			}
		}
		u32 ltot ;
		c_scan_threads( cx, looks, ltot ) ;
		if ( cx.tid == 0 )
		{
			sm->bi[0] = (int)total ;
			sm->bi[1] = 0 ;
			t4_count( cx, 2, (u64)ltot ) ;
			t4_count( cx, 3, (u64)total ) ;
			t4_count( cx, 4, (u64)total ) ;
			t4_count( cx, 5, (u64)( ( len + 3 ) / 4 ) ) ;
		}
	}
	// sequential scan along the read: equal-to-previous rule with the stale prevKmerCode semantics and the
	// >=100-postings skip rule (SeqSet.hpp:1376-1392, 1441-1455)
	else if ( cx.tid == 0 )
	{
		int skipLimit = refSet ? 0 : k / 2 ;
		u32 total = 0 ;
		int big = 0 ;
		u64 lookups = 0, postings = 0 ;
		u64 prev = 0 ; // KmerCode prevKmerCode( kmerLength ): code 0, carried from the forward into the reverse pass
		for ( int pass = 0 ; pass < 2 ; ++pass )
		{
			if ( ( pass == 0 && strand == -1 ) || ( pass == 1 && strand == 1 ) )
				continue ;
			int skipCnt = 0 ;
			for ( int q = 0 ; q < m ; ++q )
			{
				T4Pos *po = pos + pass * T4_DEV_MAX_READ + q ;
				int i = q + k - 1 ;
				if ( i == k - 1 || po->code != prev )
				{
					++lookups ;
					int size = po->cnt ;
					if ( size >= 100 && i != k - 1 && i != len - 1 )
					{
						if ( skipCnt < skipLimit )
						{
							++skipCnt ;
							continue ;
						}
					}
					if ( size >= 100 && allowTotalSkip )
						continue ;
					skipCnt = 0 ;
					if ( size > 0 )
					{
						po->base = total ;
						total += size ;
						postings += size ;
						if ( barcode == -1 && size > T4_BIG_REPEAT )
							big = 1 ;
					}
				}
				prev = po->code ;
			}
		}
		sm->bi[0] = (int)total ;
		sm->bi[1] = big ;
		t4_count( cx, 2, lookups ) ;
		t4_count( cx, 3, postings ) ;
		t4_count( cx, 4, (u64)total ) ;
		t4_count( cx, 5, (u64)( ( len + 3 ) / 4 ) ) ;
	}
	T4_SYNC() ;
	u32 H = (u32)sm->bi[0] ;
	*anyBig = sm->bi[1] ;
	T4_SYNC() ;
	c_ensure_hits( cx, H ) ;
	if ( st->error )
		return 0 ;
	u64 *keys = cx.P<u64>( st->keysAOff ) ;
	// emit.  Short lists: one thread copies the list of its own position; long lists (>= 100 postings exist)
	// are spread over the CTA with coalesced 8-byte loads.
	for ( int x = cx.tid ; x < 2 * m ; x += cx.nt )
	{
		int pass = x >= m ;
		int q = pass ? x - m : x ;
		T4Pos *po = pos + pass * T4_DEV_MAX_READ + q ;
		u32 base = po->base ;
		if ( base == 0xffffffffu )
			continue ;
		u32 cnt = po->cnt ;
		if ( anyLarge && cnt > 32 )
			continue ;
		const u64 *l = cx.P<u64>( po->listOff ) ;
		for ( u32 j = 0 ; j < cnt ; ++j )
		{
			u64 v = l[j] ;
			int idx = (int)( v >> 32 ) ;
			int off = (int)(u32)v ;
			u64 key = t4_key_of( pass ? -1 : 1, idx, q, off, 0 ) ;
			if ( barcode != -1 && t4_seq( cx, idx )->barcode != barcode )
				key = T4_KEY_INVALID ;
			keys[base + j] = key ;
		}
	}
	if ( anyLarge )
		for ( int pass = 0 ; pass < 2 ; ++pass )
			for ( int q = 0 ; q < m ; ++q )
			{
				T4Pos *po = pos + pass * T4_DEV_MAX_READ + q ;
				u32 base = po->base ;
				u32 cnt = po->cnt ;
				if ( base == 0xffffffffu || cnt <= 32 )
					continue ;
				const u64 *l = cx.P<u64>( po->listOff ) ;
				int big = ( barcode == -1 && cnt > T4_BIG_REPEAT ) ;
				for ( u32 j = cx.tid ; j < cnt ; j += cx.nt )
				{
					u64 v = l[j] ;
					int idx = (int)( v >> 32 ) ;
					int off = (int)(u32)v ;
					u64 key = t4_key_of( pass ? -1 : 1, idx, q, off, big ) ;
					if ( barcode != -1 && t4_seq( cx, idx )->barcode != barcode )
						key = T4_KEY_INVALID ;
					keys[base + j] = key ;
				}
			}
	T4_SYNC() ;
	return H ;
}

// ---------------------------------------------------------------------------
// chains: SeqSet::SortHits + GetOverlapsFromHits (SeqSet.hpp:1306, 763-1063) for novel contigs
// ---------------------------------------------------------------------------
// For novel contigs adjustRadius is 0 (SeqSet.hpp:902-904), so a candidate is a maximal run of hits on one
// diagonal; on one diagonal b and a increase together, hence LongestIncreasingSubsequence (SeqSet.hpp:342)
// returns its input unchanged and the chain IS the run.  GetVJOverlapsFromHits only ever sees isRef hits.
//
// v: the sorted hits (c_sort_hit_prefix), H valid.  keysR (may be 0): the same hits sorted in SortHits order
// (strand, idx, a, b) -- only needed to reproduce the `hits[k].repeats` indexing of SeqSet.hpp:931-947 when
// some k-mer has more than 10000 postings.
T4_D inline int c_overlaps_from_hits( T4Ctx &cx, const T4HitView &v, u32 H, const u64 *keysR, int hitLenRequired,
	int filter )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	const int k = st->kmerLength ;
	const u64 *keys = v.keys ;
	u32 *grp = v.grp ;
	u32 *run = v.run ;
	u32 *hl = v.hl ;
	u32 nG, nR ;
	c_hit_heads( cx, keys, H, grp, run, nG, nR ) ;
	// pre-pass (SeqSet.hpp:781-824), including its group-skipping loop increment, over the group heads
	if ( cx.tid == 0 )
	{
		int novelMin[2] = {3, 3} ;
		int removeOnlyRepeats[2] = {0, 0} ;
		if ( filter == 1 )
		{
			int possible[2] = {0, 0} ;
			int longest[2] = {0, 0} ;
			u32 g = 0 ;
			u32 i = 0 ;
			while ( i < H )
			{
				while ( grp[g + 1] <= i )
					++g ;
				u32 j = grp[g + 1] ;
				int plus = (int)( keys[i] >> T4_KEY_STRAND_SHIFT ) ;
				int sz = (int)( j - i ) ;
				if ( sz > novelMin[plus] )
					++possible[plus] ;
				if ( sz > longest[plus] )
					longest[plus] = sz ;
				if ( !removeOnlyRepeats[plus] )
				{
					int cnt = 0 ;
					if ( keysR == 0 )
						cnt = sz ;
					else
						for ( u32 x = i ; x < j ; ++x )
							if ( !t4_key_big( keysR[x] ) )
								++cnt ;
					if ( cnt >= novelMin[plus] )
						removeOnlyRepeats[plus] = 1 ;
				}
				i = j + 1 ; // `i = j` followed by the for-loop's ++i (SeqSet.hpp:784, 810)
			}
			for ( int s = 0 ; s <= 1 ; ++s )
			{
				if ( possible[s] > 100000 )
					novelMin[s] = (int)( longest[s] * 0.75 ) ;
				else if ( possible[s] > 10000 )
					novelMin[s] = longest[s] / 2 ;
				else if ( possible[s] > 1000 )
					novelMin[s] = longest[s] / 3 ;
				else if ( possible[s] > 100 )
					novelMin[s] = longest[s] / 4 ;
			}
		}
		sm->bi[0] = novelMin[0] ;
		sm->bi[1] = novelMin[1] ;
		sm->bi[2] = removeOnlyRepeats[0] ;
		sm->bi[3] = removeOnlyRepeats[1] ;
	}
	T4_SYNC() ;
	int novelMin[2] = { sm->bi[0], sm->bi[1] } ;
	int removeOnlyRepeats[2] = { sm->bi[2], sm->bi[3] } ;
	T4_SYNC() ;
	// one candidate per diagonal run (SeqSet.hpp:906-1057).  Every test below only rejects, so their order is free: the
	// cheap ones first.  The reference's test of the group size (< minHit) is implied by the run's, as the run lies
	// inside its group.
	for ( u32 r = cx.tid ; r < nR ; r += cx.nt )
	{
		u32 s = run[r], e = run[r + 1] ;
		hl[r] = 0 ;
		int n = (int)( e - s ) ;
		if ( n * k < hitLenRequired )
			continue ;
		u64 k0 = keys[s] ;
		int plus = (int)( k0 >> T4_KEY_STRAND_SHIFT ) ;
		if ( n < novelMin[plus] )
			continue ;
		if ( removeOnlyRepeats[plus] && keysR != 0 )
		{
			// group [gi, gj) containing this run
			u32 lo = 0, hi = nG ;
			while ( hi - lo > 1 )
			{
				u32 mid = ( lo + hi ) / 2 ;
				if ( grp[mid] <= s )
					lo = mid ;
				else
					hi = mid ;
			}
			u32 gi = grp[lo], gj = grp[lo + 1] ;
			bool hasUnique = false ;
			for ( u32 x = gi ; x < gj ; ++x )
				if ( !t4_key_big( keysR[x] ) )
				{
					hasUnique = true ;
					break ;
				}
			if ( !hasUnique )
				continue ;
			// SeqSet.hpp:931-947 indexes hits[] with the run-local range [s - gi, e - gi)
			hasUnique = false ;
			for ( u32 x = s - gi ; x < e - gi ; ++x )
				if ( !t4_key_big( keysR[x] ) )
				{
					hasUnique = true ;
					break ;
				}
			if ( !hasUnique )
				continue ;
		}
		// GetTotalHitLengthOnRead / OnSeq (SeqSet.hpp:3330, 3352): identical on a single diagonal
		int hitLen = 0 ;
		{
			u32 x = s ;
			while ( x < e )
			{
				u32 y ;
				int bx = t4_key_b( keys[x] ) ;
				int last = bx ;
				for ( y = x + 1 ; y < e ; ++y )
				{
					int by = t4_key_b( keys[y] ) ;
					if ( by > last + k - 1 )
						break ;
					last = by ;
				}
				hitLen += last - bx + k ;
				x = y ;
			}
		}
		if ( hitLen < hitLenRequired )
			continue ;
		int seqStart = t4_key_b( k0 ) ;
		int seqEnd = t4_key_b( keys[e - 1] ) + k - 1 ;
		if ( hitLen * 2 < seqEnd - seqStart + 1 )
			continue ;
		hl[r] = (u32)hitLen ;
	}
	T4_SYNC() ;
	// compact the kept runs, in key order, into overlaps
	u32 chunk = ( nR + cx.nt - 1 ) / cx.nt ;
	u32 lo = cx.tid * chunk ;
	u32 hi = lo + chunk < nR ? lo + chunk : nR ;
	if ( lo > nR )
		lo = nR ;
	u32 c = 0 ;
	for ( u32 r = lo ; r < hi ; ++r )
		if ( hl[r] )
			++c ;
	u32 total ;
	u32 o = c_scan_threads( cx, c, total ) ;
	c_ensure_ovl( cx, total ) ;
	if ( st->error )
		return 0 ;
	T4Ovl *ovl = cx.P<T4Ovl>( st->ovlOff ) ;
	for ( u32 r = lo ; r < hi ; ++r )
	{
		if ( !hl[r] )
			continue ;
		u32 s = run[r], e = run[r + 1] ;
		int hitLen = (int)hl[r] ;
		T4Ovl no ;
		no.seqIdx = t4_key_idx( keys[s] ) ;
		no.readStart = t4_key_a( keys[s] ) ;
		no.readEnd = t4_key_a( keys[e - 1] ) + k - 1 ;
		no.strand = t4_key_strand( keys[s] ) ;
		no.seqStart = t4_key_b( keys[s] ) ;
		no.seqEnd = t4_key_b( keys[e - 1] ) + k - 1 ;
		no.matchCnt = 2 * hitLen ;
		no.indelCnt = 0 ;
		no.similarity = 0 ;
		no.hcStart = (int)s ;
		no.hcCnt = (int)( e - s ) ;
		no.preMatchCnt = no.matchCnt ;
		no.infoFromHits = 0 ;
		ovl[o++] = no ;
	}
	T4_SYNC() ;
	return (int)total ;
}

// Test hook t4_test_group_hits: c_sort_hit_prefix and c_hit_heads over op->len keys given at op->read, in emission
// order.  The sorted keys go to op->out, {nG, nR, grp[0..nG], run[0..nR]} over the valid keys to op->out2.
T4_D inline void c_test_group_hits( T4Ctx &cx, T4Op *op )
{
	T4Stream *st = cx.st ;
	const u32 n = (u32)op->len ;
	c_ensure_hits( cx, n ) ;
	if ( st->error )
		return ;
	u64 *a = cx.P<u64>( st->keysAOff ) ;
	u64 *b = cx.P<u64>( st->keysBOff ) ;
	const u64 *in = t4_x<u64>( op->read ) ;
	for ( u32 i = cx.tid ; i < n ; i += cx.nt )
		a[i] = in[i] ;
	T4_SYNC() ;
	T4HitView v ;
	const u64 *sorted = c_sort_hit_prefix( cx, a, b, n, &v ) ;
	u32 c = 0 ;
	for ( u32 i = cx.tid ; i < n ; i += cx.nt )
		if ( v.keys[i] != T4_KEY_INVALID )
			++c ;
	u32 H ;
	c_scan_threads( cx, c, H ) ;
	u32 nG, nR ;
	c_hit_heads( cx, v.keys, H, v.grp, v.run, nG, nR ) ;
	u64 *out = t4_x<u64>( op->out ) ;
	int32_t *heads = t4_x<int32_t>( op->out2 ) ;
	for ( u32 i = cx.tid ; i < n ; i += cx.nt )
		out[i] = sorted[i] ;
	for ( u32 i = cx.tid ; i <= nG ; i += cx.nt )
		heads[2 + i] = (int32_t)v.grp[i] ;
	for ( u32 i = cx.tid ; i <= nR ; i += cx.nt )
		heads[3 + nG + i] = (int32_t)v.run[i] ;
	if ( cx.tid == 0 )
	{
		heads[0] = (int32_t)nG ;
		heads[1] = (int32_t)nR ;
		op->ret = (int)n ;
	}
}

// `_overlap::operator<` (SeqSet.hpp:104-128)
T4_HD inline bool t4_ovl_less( const T4Ovl &a, const T4Ovl &b )
{
	if ( a.matchCnt != b.matchCnt )
		return a.matchCnt > b.matchCnt ;
	else if ( a.similarity != b.similarity )
		return a.similarity > b.similarity ;
	else if ( a.readEnd - a.readStart != b.readEnd - b.readStart )
		return a.readEnd - a.readStart > b.readEnd - b.readStart ;
	else if ( a.seqIdx != b.seqIdx )
		return a.seqIdx < b.seqIdx ;
	else if ( a.strand != b.strand )
		return a.strand < b.strand ;
	else if ( a.readStart != b.readStart )
		return a.readStart < b.readStart ;
	else if ( a.readEnd != b.readEnd )
		return a.readEnd < b.readEnd ;
	else if ( a.seqStart != b.seqStart )
		return a.seqStart < b.seqStart ;
	else
		return a.seqEnd < b.seqEnd ;
}

// std::sort( overlaps ) with operator< (a strict total order on distinct overlaps, so any correct sort
// yields the reference's sequence).  Rank sort: n is small (tens, rarely hundreds).
T4_D inline void c_sort_overlaps( T4Ctx &cx, int n )
{
	if ( n <= 1 )
		return ;
	T4Ovl *ovl = cx.P<T4Ovl>( cx.st->ovlOff ) ;
	T4Ovl *tmp = cx.P<T4Ovl>( cx.st->ovlTmpOff ) ;
	T4_PAR_FOR( i, n )
	{
		T4Ovl me = ovl[i] ;
		int rank = 0 ;
		for ( int j = 0 ; j < n ; ++j )
		{
			if ( j == i )
				continue ;
			if ( t4_ovl_less( ovl[j], me ) || ( j < i && !t4_ovl_less( me, ovl[j] ) ) )
				++rank ;
		}
		tmp[rank] = me ;
	}
	T4_SYNC() ;
	T4_PAR_FOR( i, n )
		ovl[i] = tmp[i] ;
	T4_SYNC() ;
}

// SeqSet::IsOverlapLowComplex (SeqSet.hpp:590)
T4_D inline bool t4_low_complex( const char *r, const T4Ovl &o )
{
	int cnt[4] = {0, 0, 0, 0} ;
	for ( int i = o.readStart ; i <= o.readEnd ; ++i )
	{
		if ( r[i] == 'N' )
			continue ;
		++cnt[t4_nuc( r[i] )] ;
	}
	int lowCnt = 0, lowTotalCnt = 0 ;
	for ( int i = 0 ; i < 4 ; ++i )
		if ( cnt[i] <= 2 )
		{
			++lowCnt ;
			lowTotalCnt += cnt[i] ;
		}
	if ( lowTotalCnt * 7 >= o.readEnd - o.readStart + 1 )
		return false ;
	return lowCnt >= 2 ;
}

#if T4_CUDA
T4_D inline void c_score_all_warp( T4Ctx &cx, T4Ovl *ovl, int overlapCnt, const u64 *keys ) ;
#endif

// ---------------------------------------------------------------------------
// SeqSet::GetOverlapsFromRead (SeqSet.hpp:1508-2124), readType 0, novel contigs
// ---------------------------------------------------------------------------
// Returns the number of overlaps left in ovl[] (-1 when the read is shorter than k).
T4_D T4_BIG int c_get_overlaps( T4Ctx &cx, int len, int strand, int barcode, bool skipRepeats )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	const int k = st->kmerLength ;
	if ( len < k )
		return -1 ;
	int overlapCnt = 0 ;
	const u64 *keys = 0 ;
	for ( int pass = skipRepeats ? 0 : 1 ; pass < 2 && overlapCnt == 0 ; ++pass )
	{
		int anyBig = 0 ;
		T4_PHASE( cx, 1 ) ;
		u32 H = c_get_hits( cx, len, strand, barcode, pass == 0, &anyBig ) ;
		T4_PHASE( cx, 2 ) ;
		if ( st->error )
			return 0 ;
		u64 *a = cx.P<u64>( st->keysAOff ) ;
		u64 *b = cx.P<u64>( st->keysBOff ) ;
		const u64 *keysR = 0 ;
		if ( anyBig )
		{
			// Rare: some k-mer of the read has more than 10000 postings.  GetOverlapsFromHits then consults
			// hits[x].repeats at positions x of the SortHits order (strand, idx, readOffset, offset) -- including the
			// run-local indexing slip of SeqSet.hpp:931-947 -- so keep a second copy of the hits in that order.
			if ( H > st->hitCapR )
			{
				if ( cx.tid == 0 )
				{
					u32 nc = st->hitCapR ? st->hitCapR : 4096 ;
					while ( nc < H )
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
				T4_SYNC() ;
				if ( st->error )
					return 0 ;
			}
			u64 *ra = cx.P<u64>( st->keysROff ) ;
			u64 *rb = cx.P<u64>( st->keysR2Off ) ;
			for ( u32 i = cx.tid ; i < H ; i += cx.nt )
			{
				u64 kx = a[i] ;
				if ( kx != T4_KEY_INVALID )
					kx = ( kx & ( ~0ull << T4_KEY_IDX_SHIFT ) ) | ( (u64)t4_key_a( kx ) << 30 ) | ( (u64)t4_key_b( kx ) << 11 ) | ( kx & 1 ) ;
				ra[i] = kx ;
			}
			T4_SYNC() ;
			keysR = c_sort_keys( cx, ra, rb, H ) ;
		}
		T4HitView v ;
		keys = c_sort_hit_prefix( cx, a, b, H, &v ) ;
		// invalid keys (barcode filter) sorted to the end
		if ( barcode != -1 )
		{
			u32 c = 0 ;
			for ( u32 i = cx.tid ; i < H ; i += cx.nt )
				if ( v.keys[i] != T4_KEY_INVALID )
					++c ;
			u32 total ;
			c_scan_threads( cx, c, total ) ;
			H = total ;
		}
		T4_PHASE( cx, 3 ) ;
		overlapCnt = c_overlaps_from_hits( cx, v, H, keysR, st->hitLenRequired, pass == 0 ? 0 : 1 ) ;
		if ( st->error )
			return 0 ;
	}
	T4_PHASE( cx, 4 ) ;
	if ( overlapCnt == 0 )
		return 0 ;
	c_sort_overlaps( cx, overlapCnt ) ;
	T4Ovl *ovl = cx.P<T4Ovl>( st->ovlOff ) ;
	// keep the strand of the best overlap (SeqSet.hpp:1601-1616)
	if ( cx.tid == 0 )
	{
		int kk = 1 ;
		for ( int i = 1 ; i < overlapCnt ; ++i )
		{
			if ( ovl[i].strand != ovl[0].strand )
				continue ;
			if ( i != kk )
				ovl[kk] = ovl[i] ;
			++kk ;
		}
		sm->bi[0] = kk ;
	}
	T4_SYNC() ;
	overlapCnt = sm->bi[0] ;
	T4_SYNC() ;
	// score every overlap independently (SeqSet.hpp:1832-2020); the order-dependent pre-filters are replayed below
#if T4_CUDA
	u64 fullDps = 0 ;
	c_score_all_warp( cx, ovl, overlapCnt, keys ) ;
#else
	T4DpScratch ds = t4_dp_scratch( cx ) ;
	u64 fullDps = 0 ;
	T4_PAR_FOR( i, overlapCnt )
	{
		T4Ovl &o = ovl[i] ;
		const char *r = ( o.strand == 1 ) ? sm->read : sm->rc ;
		const u64 *hc = keys + o.hcStart ;
		int hitCnt = o.hcCnt ;
		int matchCnt = 2 * k, mismatchCnt = 0, indelCnt = 0 ;
		double similarity = 1 ;
		int *pw = t4_pw( cx, t4_seq( cx, o.seqIdx ) ) ;
		for ( int j = 1 ; j < hitCnt ; ++j )
		{
			int a0 = t4_key_a( hc[j - 1] ), a1 = t4_key_a( hc[j] ) ;
			int b0 = t4_key_b( hc[j - 1] ) ;
			// same diagonal always (see c_overlaps_from_hits)
			if ( a0 + k - 1 >= a1 )
				matchCnt += 2 * ( a1 - a0 ) ;
			else
			{
				matchCnt += 2 * k ;
				int gap = a1 - ( a0 + k ) ;
				if ( gap > st->nomatchGapLimit )
				{
					similarity = 0 ;
					break ;
				}
				int full = 0 ;
				t4_dp_equal( pw + 4 * ( b0 + k ), r + a0 + k, gap, ds.align, (u32 *)ds.act, false, &full ) ;
				fullDps += full ;
				int cnt0, cnt1, cnt2 ;
				t4_align_stats( ds.align, false, cnt0, cnt1, cnt2 ) ;
				matchCnt += 2 * cnt0 ;
				mismatchCnt += cnt1 ;
				indelCnt += cnt2 ;
				if ( indelCnt > 0 )
				{
					similarity = 0 ;
					break ;
				}
			}
		}
		o.preMatchCnt = o.matchCnt ;
		o.matchCnt = matchCnt ;
		o.indelCnt = indelCnt ;
		if ( similarity == 1 )
			o.similarity = (double)matchCnt / ( o.seqEnd - o.seqStart + 1 + o.readEnd - o.readStart + 1 ) ;
		else
			o.similarity = 0 ;
		if ( t4_low_complex( r, o ) )
			o.similarity = 0 ;
	}
#endif
	if ( fullDps )
		t4_count( cx, 7, fullDps ) ;
	t4_count( cx, 6, cx.tid == 0 ? (u64)overlapCnt : 0 ) ;
	T4_SYNC() ;
	// sequential replay of the loop's bookkeeping: infoFromHits, bestNovelOverlap pre-filters (only when
	// overlapCnt > 50), final similarity filter (SeqSet.hpp:1673-1794, 2024-2118)
	if ( cx.tid == 0 )
	{
		int best = -1 ;
		int radius = st->radius ;
		for ( int i = 0 ; i < overlapCnt ; ++i )
		{
			T4Ovl &o = ovl[i] ;
			o.infoFromHits = i ;
			bool filtered = false ;
			if ( best != -1 && overlapCnt > 50 )
			{
				T4Ovl &bo = ovl[best] ;
				int pm = o.preMatchCnt ;
				if ( bo.readStart == 0 && bo.readEnd == len - 1 )
				{
					if ( bo.similarity == 1 )
						filtered = true ;
					else if ( bo.similarity > st->repeatSimilarity && pm < 0.9 * bo.matchCnt )
						filtered = true ;
				}
				if ( !filtered && bo.readStart + len - 1 - bo.readEnd < radius )
				{
					if ( bo.similarity == 1 && pm < 0.9 * bo.matchCnt )
						filtered = true ;
					else if ( ( bo.similarity > st->repeatSimilarity || st->isLongSeqSet ) && pm < 0.8 * bo.matchCnt )
						filtered = true ;
				}
				if ( !filtered && o.seqStart - o.readStart >= radius
					&& o.seqEnd + ( len - 1 - o.readEnd ) + radius < t4_seq( cx, o.seqIdx )->len
					&& bo.matchCnt > 0.97 * ( 2 * len )
					&& bo.similarity > st->repeatSimilarity
					&& pm < 0.9 * bo.matchCnt )
					filtered = true ;
				if ( !filtered && pm < 0.4 * bo.matchCnt )
					filtered = true ;
				if ( !filtered && overlapCnt > 1000 && pm < 0.9 * bo.matchCnt )
					filtered = true ;
			}
			if ( filtered )
			{
				o.similarity = 0 ;
				o.matchCnt = o.preMatchCnt ;
				o.indelCnt = 0 ;
				continue ;
			}
			if ( o.similarity > 0 )
			{
				if ( best == -1 || t4_ovl_less( o, ovl[best] ) )
					best = i ;
			}
		}
		int kk = 0 ;
		for ( int i = 0 ; i < overlapCnt ; ++i )
		{
			if ( ovl[i].similarity < st->novelSeqSimilarity )
				continue ;
			if ( kk != i )
				ovl[kk] = ovl[i] ;
			++kk ;
		}
		sm->bi[0] = kk ;
	}
	T4_SYNC() ;
	overlapCnt = sm->bi[0] ;
	T4_SYNC() ;
	return overlapCnt ;
}

// ---------------------------------------------------------------------------
// SeqSet::ExtendOverlap (SeqSet.hpp:1165-1277).  Pure function of (read, contig, overlap).
// ---------------------------------------------------------------------------
struct T4AlignView      // an edit string either as an explicit array (full DP) or as match bits (all-diagonal alignment)
{
	const signed char *a ;
	const u32 *bits ;
	int n ;
	int dp ;
	T4_D inline int get( int i ) const
	{
		if ( a )
			return a[i] ;
		return ( ( bits[i >> 5] >> ( i & 31 ) ) & 1 ) ? EDIT_MATCH : EDIT_MISMATCH ;
	}
} ;

// GlobalAlignment_PosWeight for an overhang of equal lengths n whose IsBaseEqual outcomes are given as bits:
// the trivial cases and the <= 2 mismatch fast path (AlignAlgo.hpp:59-103) need no DP at all.
T4_D inline T4AlignView t4_overhang_align( const int *tw, const char *p, int n, const u32 *bits, T4DpScratch &ds )
{
	T4AlignView v ;
	v.a = 0 ;
	v.bits = bits ;
	v.n = n ;
	v.dp = 0 ;
	if ( n <= 1 )
		return v ;
	int matches = 0 ;
	for ( int w = 0 ; w * 32 < n ; ++w )
	{
		u32 x = bits[w] ;
		if ( ( w + 1 ) * 32 > n )
			x &= ( 1u << ( n - w * 32 ) ) - 1u ;
#if T4_CUDA
		matches += __popc( x ) ;
#else
		matches += __builtin_popcount( x ) ;
#endif
	}
	int score = SCORE_MATCH * matches + SCORE_MISMATCH * ( n - matches ) ;
	if ( score >= n * SCORE_MATCH + 2 * SCORE_INDEL )
		return v ;
	t4_dp_equal( tw, p, n, ds.align, (u32 *)ds.act, true, 0 ) ;
	v.dp = 1 ;
	v.a = ds.align ;
	v.bits = 0 ;
	int l = 0 ;
	while ( ds.align[l] != -1 )
		++l ;
	v.n = l ;
	return v ;
}

struct T4SideStats { int m, x, ind, good ; } ;

// Statistics ExtendOverlap takes from one overhang alignment (SeqSet.hpp:1176-1224): edit counts over the whole
// string, and the longest prefix (seen from the anchor: fromEnd for the left overhang) of match/mismatch ops whose
// running match fraction exceeds 0.75 at a match.
T4_D inline T4SideStats t4_side_stats( const T4AlignView &av, bool fromEnd )
{
	T4SideStats r ;
	r.m = r.x = r.ind = r.good = 0 ;
	for ( int i = 0 ; i < av.n ; ++i )
	{
		int e = av.get( i ) ;
		if ( e == EDIT_MATCH )
			++r.m ;
		else if ( e == EDIT_MISMATCH )
			++r.x ;
		else
			++r.ind ;
	}
	int tmpMatchCnt = 0 ;
	for ( int kk = 0 ; kk < av.n ; ++kk )
	{
		int e = av.get( fromEnd ? av.n - 1 - kk : kk ) ;
		if ( e == EDIT_MATCH )
		{
			++tmpMatchCnt ;
			if ( tmpMatchCnt > 0.75 * ( kk + 1 ) )
				r.good = kk + 1 ;
		}
		else if ( e != EDIT_MISMATCH )
			break ;
	}
	return r ;
}

// One overhang side of ExtendOverlap (SeqSet.hpp:1165-1175): n columns from contig column col against read positions
// rp .. rp + n - 1.  The only place that derives a side from an overlap.
struct T4Side { int n, col, rp ; } ;

// Side `right` (0 left, 1 right) of overlap o of a read of length len against a contig of length seqLen.
T4_HD inline T4Side t4_overhang_side( const T4Ovl &o, int right, int len, int seqLen )
{
	T4Side s ;
	if ( !right )
	{
		s.n = t4_min( o.readStart, o.seqStart ) ;
		s.col = o.seqStart - s.n ;
		s.rp = o.readStart - s.n ;
	}
	else
	{
		s.n = t4_min( len - 1 - o.readEnd, seqLen - 1 - o.seqEnd ) ;
		s.col = o.seqEnd + 1 ;
		s.rp = o.readEnd + 1 ;
	}
	return s ;
}

// The rest of ExtendOverlap (SeqSet.hpp:1226-1277) given both sides' statistics.
T4_D inline int t4_extend_finish( T4Ctx &cx, int len, T4Contig *seq, double mismatchThresholdFactor, const T4Ovl &overlap, T4Ovl &ext,
	const T4SideStats &ls, const T4SideStats &rs )
{
	T4Stream *st = cx.st ;
	int ret = 1 ;
	int leftOverhangSize = t4_overhang_side( overlap, 0, len, seq->len ).n ;
	int rightOverhangSize = t4_overhang_side( overlap, 1, len, seq->len ).n ;
	int matchCnt = ls.m + rs.m, mismatchCnt = ls.x + rs.x ;
	if ( ls.ind > 0 )
	{
		leftOverhangSize = 0 ;
		ret = 0 ;
	}
	if ( rs.ind > 0 )
	{
		rightOverhangSize = 0 ;
		ret = 0 ;
	}
	int goodLeftOverhangSize = ls.good, goodRightOverhangSize = rs.good ;
	int mismatchThreshold = 2 ;
	if ( leftOverhangSize >= 2 )
		++mismatchThreshold ;
	if ( rightOverhangSize >= 2 )
		++mismatchThreshold ;
	double densityThreshold = 1.5 / st->kmerLength ;
	mismatchThreshold = (int)( mismatchThreshold * mismatchThresholdFactor ) ;
	if ( mismatchCnt > mismatchThreshold && (double)mismatchCnt / ( leftOverhangSize + rightOverhangSize ) > densityThreshold )
		ret = 0 ;
	ext = overlap ;
	ext.readStart = overlap.readStart - leftOverhangSize ;
	ext.readEnd = overlap.readEnd + rightOverhangSize ;
	ext.seqStart = overlap.seqStart - leftOverhangSize ;
	ext.seqEnd = overlap.seqEnd + rightOverhangSize ;
	ext.matchCnt = 2 * matchCnt + overlap.matchCnt ;
	ext.similarity = (double)( 2 * matchCnt + overlap.matchCnt ) /
		( ext.readEnd - ext.readStart + 1 + ext.seqEnd - ext.seqStart + 1 ) ;
	// only seqIdx, coordinates, strand, matchCnt, similarity are assigned by the reference; the remaining
	// fields of the destination keep whatever they held.  None of them is observable afterwards.
	if ( ext.similarity < st->novelSeqSimilarity )
	{
		ext = overlap ;
		ret = 0 ;
	}
	if ( ret == 0 )
	{
		ext.readStart = overlap.readStart - goodLeftOverhangSize ;
		ext.readEnd = overlap.readEnd + goodRightOverhangSize ;
		ext.seqStart = overlap.seqStart - goodLeftOverhangSize ;
		ext.seqEnd = overlap.seqEnd + goodRightOverhangSize ;
	}
	return ret ;
}

// lbits / rbits: IsBaseEqual( posWeight column, read base ) for the left / right overhang, bit t = t-th overhang position
T4_D inline int t4_extend_overlap( T4Ctx &cx, const char *r, int len, T4Contig *seq, double mismatchThresholdFactor,
	T4DpScratch &ds, const T4Ovl &overlap, T4Ovl &ext, const u32 *lbits, const u32 *rbits )
{
	const T4Side L = t4_overhang_side( overlap, 0, len, seq->len ), R = t4_overhang_side( overlap, 1, len, seq->len ) ;
	int *pw = t4_pw( cx, seq ) ;
	T4SideStats ls, rs ;
	{
		T4AlignView av = t4_overhang_align( pw + 4 * L.col, r + L.rp, L.n, lbits, ds ) ;
		if ( av.dp )
			t4_count( cx, 1, 1 ) ;
		ls = t4_side_stats( av, true ) ;
	}
	{
		T4AlignView av = t4_overhang_align( pw + 4 * R.col, r + R.rp, R.n, rbits, ds ) ;
		if ( av.dp )
			t4_count( cx, 1, 1 ) ;
		rs = t4_side_stats( av, false ) ;
	}
	return t4_extend_finish( cx, len, seq, mismatchThresholdFactor, overlap, ext, ls, rs ) ;
}

#if T4_CUDA
// ---------------------------------------------------------------------------
// warp-cooperative forms (product build only; the emulation uses the sequential forms above, and the GPU parity
// tests compare these against the reference)
// ---------------------------------------------------------------------------
#define T4_FULL 0xffffffffu

// Banded DP for equal lengths in a HALF warp: the 16 lanes own the 13 window slots, anti-diagonal schedule
// T = 2 i + slot (cell (i, slot) needs (i-1, slot) at T-2 and (i, slot-1), (i-1, slot+1) at T-1, which are the
// neighbours' most recent values, exchanged by shuffles).  All 32 lanes call; a half with n == 0 idles.
// nib: the IsBaseEqual nibbles of the n target columns, 8 per word (staged in shared memory by w_stage_side), so the
// loop touches no global memory.  actBase / actStride: traceback words of slot s at actBase + s * actStride.
// Returns the score in every lane of the half; the half's lane 0 writes the edit string to `align`; *alignLen = its length.
T4_D inline int w_dp_equal_half( T4Ctx &cx, const u32 *nib, const char *p, int n, signed char *alignBuf, int alignCap, int *alignLen,
	u32 *actBase, int actStride )
{
	const int lane = cx.tid & 31, hl = lane & 15 ;
	const int nmax = max( n, __shfl_xor_sync( T4_FULL, n, 16 ) ) ;
	const int negInf = ( n + 1 ) * ( n + 1 ) * SCORE_INDEL ;
	const int j0 = hl - 6 ;
	int latest = ( j0 == 0 ) ? 0 : ( j0 > 0 ? SCORE_INDEL + j0 * SCORE_INDEL : negInf ) ;
	u32 *myAct = actBase + hl * actStride ;
	u32 aw = 0 ;
	for ( int T = 2 ; T <= 2 * nmax + 12 ; ++T )
	{
		int vl = __shfl_up_sync( T4_FULL, latest, 1, 16 ) ;
		int vu = __shfl_down_sync( T4_FULL, latest, 1, 16 ) ;
		int i = ( T - hl ) >> 1 ;
		if ( hl < 13 && ( ( T - hl ) & 1 ) == 0 && i >= 1 && i <= n )
		{
			int j = i - 6 + hl ;
			int start = i - 5 < 1 ? 1 : i - 5 ;
			int end = i + 5 > n ? n : i + 5 ;
			int val ;
			u32 a = 0 ;
			if ( j == 0 )
				val = SCORE_INDEL + i * SCORE_INDEL ;
			else if ( j < start || j > end )
				val = negInf ;
			else
			{
				char pc = p[i - 1] ;
				u32 nb = ( nib[( j - 1 ) >> 3] >> ( 4 * ( ( j - 1 ) & 7 ) ) ) & 15u ;
				bool eq = ( pc == 'N' ) || ( ( nb >> t4_nuc( pc ) ) & 1u ) ;
				int diff = eq ? SCORE_MATCH : SCORE_MISMATCH ;
				int dg = latest + diff, lf = vl + SCORE_INDEL, up = vu + SCORE_INDEL ;
				val = dg ;
				if ( lf > val ) val = lf ;
				if ( up > val ) val = up ;
				if ( lf == val ) a = EDIT_DELETE ;
				if ( up == val ) a = EDIT_INSERT ;
				if ( dg == val ) a = eq ? EDIT_MATCH : EDIT_MISMATCH ;
			}
			aw |= a << ( 2 * ( i & 15 ) ) ;
			if ( ( i & 15 ) == 15 || i == n )
			{
				myAct[i >> 4] = aw ;
				aw = 0 ;
			}
			latest = val ;
		}
	}
	int ret = __shfl_sync( T4_FULL, latest, 6, 16 ) ;
	__syncwarp() ;
	int tag = 0 ;
	if ( hl == 0 && n > 0 )
	{
		// the edit string is written from the end of the buffer towards its start: it ends up in reading order at
		// alignBuf + alignCap - 1 - tag without a reversal pass
		signed char *align = alignBuf + alignCap - 1 ;
		*align = -1 ;
		int tagi = n, tagj = n ;
		while ( tagi > 0 || tagj > 0 )
		{
			int a ;
			if ( tagi > 0 && tagj > 0 )
			{
				int slot = tagj - ( tagi - 6 ) ;
				a = (int)( ( actBase[slot * actStride + ( tagi >> 4 )] >> ( 2 * ( tagi & 15 ) ) ) & 3u ) ;
			}
			else if ( tagj > 0 )
				a = ( tagj >= 2 ) ? EDIT_DELETE : EDIT_MATCH ;
			else
				a = ( tagi >= 2 ) ? EDIT_INSERT : EDIT_MATCH ;
			++tag ;
			align[-tag] = (signed char)a ;
			if ( a == EDIT_DELETE )
				--tagj ;
			else if ( a == EDIT_INSERT )
				--tagi ;
			else
			{
				--tagi ;
				--tagj ;
			}
		}
	}
	tag = __shfl_sync( T4_FULL, tag, 0, 16 ) ;
	__syncwarp() ;
	*alignLen = tag ;
	return ret ;
}

// Stage one side for a warp: the n columns with equality bytes te[0..n) (t4_eq) against p[0..n): IsBaseEqual
// nibbles (8 per word) and the match bits, into shared memory.  Returns the number of matches.
T4_D inline int w_stage_side( const unsigned char *te, const char *p, int n, u32 *nibOut, u32 *bitsOut, int lane )
{
	int matches = 0 ;
	for ( int t0 = 0 ; t0 < n ; t0 += 32 )
	{
		int t = t0 + lane ;
		u32 nb = 0 ;
		bool eq = false ;
		if ( t < n )
		{
			nb = te[t] ;
			char pc = p[t] ;
			eq = ( pc == 'N' ) || ( ( nb >> t4_nuc( pc ) ) & 1u ) ;
		}
		u32 v = nb << ( 4 * ( lane & 7 ) ) ;
		v |= __shfl_xor_sync( T4_FULL, v, 1 ) ;
		v |= __shfl_xor_sync( T4_FULL, v, 2 ) ;
		v |= __shfl_xor_sync( T4_FULL, v, 4 ) ;
		if ( ( lane & 7 ) == 0 )
			nibOut[( t0 >> 3 ) + ( lane >> 3 )] = v ;
		u32 mb = __ballot_sync( T4_FULL, eq ) ;
		if ( lane == 0 )
			bitsOut[t0 >> 5] = mb ;
		matches += __popc( mb ) ;
	}
	__syncwarp() ;
	return matches ;
}

// t4_side_stats with all 32 lanes (ballots / popcounts).  Identical in every lane.
T4_D inline T4SideStats w_side_stats( const T4AlignView &v, bool fromEnd, int lane )
{
	T4SideStats r ;
	r.m = r.x = r.ind = r.good = 0 ;
	int mbase = 0 ;
	bool stopped = false ;
	for ( int base = 0 ; base < v.n ; base += 32 )
	{
		int kk = base + lane ;
		int e = -1 ;
		if ( kk < v.n )
			e = v.get( fromEnd ? v.n - 1 - kk : kk ) ;
		unsigned mb = __ballot_sync( T4_FULL, e == EDIT_MATCH ) ;
		unsigned xb = __ballot_sync( T4_FULL, e == EDIT_MISMATCH ) ;
		unsigned ib = __ballot_sync( T4_FULL, e == EDIT_INSERT || e == EDIT_DELETE ) ;
		r.m += __popc( mb ) ;
		r.x += __popc( xb ) ;
		r.ind += __popc( ib ) ;
		if ( !stopped )
		{
			unsigned le = ( lane == 31 ) ? 0xffffffffu : ( ( 1u << ( lane + 1 ) ) - 1u ) ;
			int mk = mbase + __popc( mb & le ) ;
			bool cond = ( e == EDIT_MATCH ) && ( ( ib & le ) == 0 ) && ( mk > 0.75 * ( kk + 1 ) ) ;
			unsigned cb = __ballot_sync( T4_FULL, cond ) ;
			if ( cb )
				r.good = base + ( 31 - __clz( cb ) ) + 1 ;
			if ( ib )
				stopped = true ;
			mbase += __popc( mb ) ;
		}
	}
	return r ;
}

// One overhang side of w_side_pair: n columns with equality bytes te[0..n) against p[0..n) (n == 0: no side); fromEnd
// for a left overhang.  act / actStride: the traceback words of its half-warp DP; al / alCap: its edit-string buffer.
struct T4DpSide
{
	const unsigned char *te ;
	const char *p ;
	int n ;
	bool fromEnd ;
	u32 *act ;
	int actStride ;
	signed char *al ;
	int alCap ;
} ;

// Two overhang alignments on one warp: both sides are staged, side h runs w_dp_equal_half on half-warp h (both halves
// at once), then the whole warp takes each side's statistics from its edit string.  Results identical in every lane.
T4_D inline void w_side_pair( T4Ctx &cx, const T4DpSide &s0, const T4DpSide &s1, u32 ( *nib )[64], u32 ( *bits )[16],
	T4SideStats &r0, T4SideStats &r1 )
{
	const int lane = cx.tid & 31 ;
	w_stage_side( s0.te, s0.p, s0.n, nib[0], bits[0], lane ) ;
	w_stage_side( s1.te, s1.p, s1.n, nib[1], bits[1], lane ) ;
	const bool hi = lane >= 16 ;
	int alen = 0 ;
	w_dp_equal_half( cx, nib[hi ? 1 : 0], hi ? s1.p : s0.p, hi ? s1.n : s0.n, hi ? s1.al : s0.al, hi ? s1.alCap : s0.alCap, &alen,
		hi ? s1.act : s0.act, hi ? s1.actStride : s0.actStride ) ;
	const int a0 = __shfl_sync( T4_FULL, alen, 0 ), a1 = __shfl_sync( T4_FULL, alen, 16 ) ;
	T4AlignView v ;
	v.bits = 0 ;
	v.dp = 1 ;
	v.a = s0.al + s0.alCap - 1 - a0 ;
	v.n = a0 ;
	r0 = w_side_stats( v, s0.fromEnd, lane ) ;
	v.a = s1.al + s1.alCap - 1 - a1 ;
	v.n = a1 ;
	r1 = w_side_stats( v, s1.fromEnd, lane ) ;
}

T4_D inline signed char *t4_align_of_thread( T4Ctx &cx, int tid )
{
	return (signed char *)( cx.P<char>( cx.st->dpOff ) + (size_t)tid * cx.st->dpStride + 2 * T4_DP_W * 4 + 8
		+ ( T4_DEV_MAX_READ + 1 ) * T4_DP_W + 8 ) ;
}

// Overlap scoring (SeqSet.hpp:1832-2020) for every overlap: one warp per overlap, lanes over consecutive hit pairs.
// A failed overlap (gap over the limit, or an indel in a gap) gets similarity 0; its counts are unobservable.
T4_D inline void c_score_all_warp( T4Ctx &cx, T4Ovl *ovl, int overlapCnt, const u64 *keys )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	const int k = st->kmerLength ;
	const int warp = cx.tid >> 5, nwarps = cx.nt >> 5, lane = cx.tid & 31 ;
	u64 fullDps = 0 ;
	for ( int i = warp ; i < overlapCnt ; i += nwarps )
	{
		const T4Ovl o = ovl[i] ;
		const char *r = ( o.strand == 1 ) ? sm->read : sm->rc ;
		const u64 *hc = keys + o.hcStart ;
		const int hitCnt = o.hcCnt ;
		const unsigned char *eqb = t4_eq( cx, t4_seq( cx, o.seqIdx ) ) ;
		int acc = 0 ;           // per-lane partial of matchCnt
		bool fail = false ;
		for ( int base = 1 ; base < hitCnt && !fail ; base += 32 )
		{
			int j = base + lane ;
			int a0 = 0, a1 = 0, b0 = 0 ;
			bool gapHere = false ;
			if ( j < hitCnt )
			{
				u64 k0 = hc[j - 1], k1 = hc[j] ;
				a0 = t4_key_a( k0 ) ; a1 = t4_key_a( k1 ) ; b0 = t4_key_b( k0 ) ;
				if ( a0 + k - 1 >= a1 )
					acc += 2 * ( a1 - a0 ) ;
				else
				{
					acc += 2 * k ;
					gapHere = true ;
				}
			}
			unsigned gb = __ballot_sync( T4_FULL, gapHere ) ;
			while ( gb && !fail )
			{
				int src = __ffs( gb ) - 1 ;
				gb &= gb - 1 ;
				int ga0 = __shfl_sync( T4_FULL, a0, src ), ga1 = __shfl_sync( T4_FULL, a1, src ), gb0 = __shfl_sync( T4_FULL, b0, src ) ;
				int gap = ga1 - ( ga0 + k ) ;
				if ( gap > st->nomatchGapLimit )
				{
					fail = true ;
					break ;
				}
				const char *p = r + ga0 + k ;
				// IsBaseEqual along the diagonal of the gap (nibbles + match bits staged in shared memory)
				int matches = w_stage_side( eqb + gb0 + k, p, gap, sm->wnib[warp][0], sm->wbits[warp][0], lane ) ;
				int cnt0 = matches ;
				if ( gap >= 2 && SCORE_MATCH * matches + SCORE_MISMATCH * ( gap - matches ) < gap * SCORE_MATCH + 2 * SCORE_INDEL )
				{
					int alen = 0 ;
					bool small = gap < 16 * T4_WACT_WORDS ;
					u32 *actBase = small ? sm->wact[warp][lane < 16 ? 0 : 1] : (u32 *)t4_dp_scratch_of( cx, ( cx.tid & ~15 ) ).act ;
					int actStride = small ? T4_WACT_WORDS : (int)( T4_DP_STRIDE / 4 ) ;
					signed char *abuf = small ? sm->wal[warp][lane < 16 ? 0 : 1] : t4_align_of_thread( cx, cx.tid & ~15 ) ;
					int acap = small ? (int)sizeof( sm->wal[0][0] ) : 2 * T4_DEV_MAX_READ + 8 ;
					w_dp_equal_half( cx, sm->wnib[warp][0], p, lane < 16 ? gap : 0, abuf, acap, &alen, actBase, actStride ) ;
					alen = __shfl_sync( T4_FULL, alen, 0 ) ;
					++fullDps ;
					signed char *buf0 = small ? sm->wal[warp][0] : t4_align_of_thread( cx, warp * 32 ) ;
					T4AlignView v ;
					v.a = buf0 + acap - 1 - alen ; v.bits = 0 ; v.n = alen ; v.dp = 1 ;
					T4SideStats ss = w_side_stats( v, false, lane ) ;
					cnt0 = ss.m ;
					if ( ss.ind > 0 )
						fail = true ;
				}
				if ( lane == 0 )
					acc += 2 * cnt0 ;
			}
		}
		int matchCnt = 2 * k + __reduce_add_sync( T4_FULL, acc ) ;
		// IsOverlapLowComplex (SeqSet.hpp:590)
		int c0 = 0, c1 = 0, c2 = 0, c3 = 0 ;
		for ( int t0 = o.readStart ; t0 <= o.readEnd ; t0 += 32 )
		{
			int t = t0 + lane ;
			int x = -1 ;
			if ( t <= o.readEnd && r[t] != 'N' )
				x = t4_nuc( r[t] ) ;
			c0 += __popc( __ballot_sync( T4_FULL, x == 0 ) ) ;
			c1 += __popc( __ballot_sync( T4_FULL, x == 1 ) ) ;
			c2 += __popc( __ballot_sync( T4_FULL, x == 2 ) ) ;
			c3 += __popc( __ballot_sync( T4_FULL, x == 3 ) ) ;
		}
		if ( lane == 0 )
		{
			T4Ovl &w = ovl[i] ;
			w.preMatchCnt = o.matchCnt ;
			w.matchCnt = matchCnt ;
			w.indelCnt = 0 ;
			double sim = 0 ;
			if ( !fail )
				sim = (double)matchCnt / ( o.seqEnd - o.seqStart + 1 + o.readEnd - o.readStart + 1 ) ;
			int cnt[4] = { c0, c1, c2, c3 } ;
			int lowCnt = 0, lowTotalCnt = 0 ;
			for ( int x = 0 ; x < 4 ; ++x )
				if ( cnt[x] <= 2 )
				{
					++lowCnt ;
					lowTotalCnt += cnt[x] ;
				}
			if ( !( lowTotalCnt * 7 >= o.readEnd - o.readStart + 1 ) && lowCnt >= 2 )
				sim = 0 ;
			w.similarity = sim ;
		}
		__syncwarp() ;
	}
	if ( lane == 0 && fullDps )
		t4_count( cx, 7, fullDps ) ;
}
#endif

// ---------------------------------------------------------------------------
// gene names
// ---------------------------------------------------------------------------
// SeqSet::GetChainType (SeqSet.hpp:5132)
T4_D inline int t4_chain_type( const char *name )
{
	if ( name[0] == 'I' )
	{
		if ( name[2] == 'H' ) return 0 ;
		else if ( name[2] == 'K' ) return 1 ;
		else if ( name[2] == 'L' ) return 2 ;
	}
	else if ( name[0] == 'T' )
	{
		if ( name[2] == 'A' ) return 3 ;
		else if ( name[2] == 'B' ) return 4 ;
		else if ( name[2] == 'G' ) return 5 ;
		else if ( name[2] == 'D' ) return 6 ;
	}
	return 8 ;
}

// SeqSet::GetGeneType (SeqSet.hpp:5076) on name[0..n)
T4_D inline int t4_gene_type( const char *name, int n )
{
	// the reference reads name[3], name[4] of a NUL-terminated string; positions past the end read as '\0'
	char c0 = n > 0 ? name[0] : 0, c1 = n > 1 ? name[1] : 0, c3 = n > 3 ? name[3] : 0, c4 = n > 4 ? name[4] : 0 ;
	if ( c0 == 'N' && c1 == 'o' )
		return -1 ;
	switch ( c3 )
	{
		case 'V': return 0 ;
		case 'D': return ( c4 >= '0' && c4 <= '9' ) ? 1 : 3 ;
		case 'J': return 2 ;
		case 'L':
		{
			char tmp[3] = { c0, c1, n > 2 ? name[2] : (char)0 } ;
			if ( t4_chain_type( tmp ) == 2 )
				return -1 ;
			return 3 ;
		}
		default: return 3 ;
	}
}

// SeqSet::IsNameCompatible (SeqSet.hpp:3374): b comes after a
T4_D inline bool t4_name_compatible( const char *a, int na, const char *b, int nb )
{
	int maxA = -1, minB = 10 ;
	int i, j ;
	for ( i = 0 ; i < na ; )
	{
		if ( a[i] == '+' )
		{
			++i ;
			continue ;
		}
		for ( j = i ; j < na && a[j] != '+' ; ++j )
			;
		int gt = t4_gene_type( a + i, j - i ) ;
		if ( gt > maxA )
			maxA = gt ;
		i = j ;
	}
	for ( i = 0 ; i < nb ; )
	{
		if ( b[i] == '+' )
		{
			++i ;
			continue ;
		}
		for ( j = i ; j < nb && b[j] != '+' ; ++j )
			;
		int gt = t4_gene_type( b + i, j - i ) ;
		if ( gt < minB && gt != -1 )
			minB = gt ;
		i = j ;
	}
	return maxA <= minB ;
}

T4_D inline bool t4_name_eq( const char *a, int na, const char *b, int nb )
{
	if ( na != nb )
		return false ;
	for ( int i = 0 ; i < na ; ++i )
		if ( a[i] != b[i] )
			return false ;
	return true ;
}

// ---------------------------------------------------------------------------
// consensus maintenance
// ---------------------------------------------------------------------------
// SeqSet::SubstituteConsensusPos (SeqSet.hpp:11058), updateIndex = true
T4_D inline void s_substitute_consensus_pos( T4Ctx &cx, int seqIdx, int pos, char c )
{
	T4Contig *seq = t4_seq( cx, seqIdx ) ;
	char *cons = t4_cons( cx, seq ) ;
	if ( pos >= seq->len || cons[pos] == c )
		return ;
	int kl = cx.st->kmerLength ;
	int start = pos - kl + 1 ;
	int end = pos + kl - 1 ;
	if ( start < 0 )
		start = 0 ;
	if ( end >= seq->len )
		end = seq->len - 1 ;
	s_remove_index( cx, cons + start, end - start + 1, seqIdx, seq->barcode, start ) ;
	cons[pos] = c ;
	s_build_index( cx, cons + start, end - start + 1, seqIdx, seq->barcode, start ) ;
}

// SeqSet::SubstituteConsensusPos, collective variant
T4_D inline void c_substitute_consensus_pos( T4Ctx &cx, int seqIdx, int pos, char c )
{
	T4Contig *seq = t4_seq( cx, seqIdx ) ;
	char *cons = t4_cons( cx, seq ) ;
	T4_SYNC() ;
	bool skip = ( pos >= seq->len || cons[pos] == c ) ;
	T4_SYNC() ;
	if ( skip )
		return ;
	int kl = cx.st->kmerLength ;
	int start = pos - kl + 1 ;
	int end = pos + kl - 1 ;
	if ( start < 0 )
		start = 0 ;
	if ( end >= seq->len )
		end = seq->len - 1 ;
	c_index_op( cx, cons + start, end - start + 1, T4_IDX_REMOVE, seqIdx, seq->barcode, start, 0 ) ;
	if ( cx.tid == 0 )
		cons[pos] = c ;
	T4_SYNC() ;
	c_index_op( cx, cons + start, end - start + 1, T4_IDX_BUILD, seqIdx, seq->barcode, start, 0 ) ;
}

// SeqSet::UpdateConsensus (SeqSet.hpp:4537-4588).  Serial.
T4_D inline void s_update_consensus( T4Ctx &cx, int seqIdx, bool updateIndex )
{
	T4Contig *seq = t4_seq( cx, seqIdx ) ;
	char *cons = t4_cons( cx, seq ) ;
	int *pw = t4_pw( cx, seq ) ;
	int changes = 0 ;
	for ( int pass = 0 ; pass < 2 ; ++pass )
	{
		// pass 0 counts; pass 1 (after the index removal) applies -- the reference collects a change list first
		for ( int i = 0 ; i < seq->len ; ++i )
		{
			int max = 0, maxTag = 0 ;
			for ( int j = 0 ; j < 4 ; ++j )
				if ( pw[4 * i + j] > max )
				{
					max = pw[4 * i + j] ;
					maxTag = j ;
				}
			if ( max == 0 )
				continue ;
			int cur = t4_nuc( cons[i] ) ;
			if ( cur != maxTag && pw[4 * i + cur] < max )
			{
				if ( pass == 0 )
					++changes ;
				else
					cons[i] = t4_numToNuc( maxTag ) ;
			}
		}
		if ( pass == 0 )
		{
			if ( changes == 0 )
				return ;
			if ( updateIndex )
				s_remove_index( cx, cons, seq->len, seqIdx, seq->barcode, 0 ) ;
		}
	}
	if ( updateIndex )
		s_build_index( cx, cons, seq->len, seqIdx, seq->barcode, 0 ) ;
}

// SeqSet::UpdateAllConsensus (SeqSet.hpp:4525).  Collective: contigs are scanned in parallel, the rare
// contigs that change are fixed up serially in slot order.
T4_D T4_BIG void c_update_all_consensus( T4Ctx &cx )
{
	T4Stream *st = cx.st ;
	T4_SYNC() ;
	// Order matters only through the index multiset, which is order independent; changed contigs are
	// processed by thread 0 in slot order like the reference.
	u32 *flag = cx.P<u32>( st->grpOff ) ; // scratch, hitCap + 1 entries; fall back to serial when too small
	bool useFlags = (u32)st->nSeqs <= st->hitCap ;
	if ( useFlags )
	{
		T4_PAR_FOR( s, st->nSeqs )
		{
			T4Contig *seq = t4_seq( cx, s ) ;
			u32 f = 0 ;
			if ( seq->consOff != 0 && !( seq->flags & T4_CF_NOINDEX ) ) // purged: `if (seq.posWeightCompressed) return` (SeqSet.hpp:4542)
			{
				const char *cons = t4_cons( cx, seq ) ;
				const int *pw = t4_pw( cx, seq ) ;
				for ( int i = 0 ; i < seq->len && !f ; ++i )
				{
					int max = 0, maxTag = 0 ;
					for ( int j = 0 ; j < 4 ; ++j )
						if ( pw[4 * i + j] > max )
						{
							max = pw[4 * i + j] ;
							maxTag = j ;
						}
					if ( max == 0 )
						continue ;
					int cur = t4_nuc( cons[i] ) ;
					if ( cur != maxTag && pw[4 * i + cur] < max )
						f = 1 ;
				}
			}
			flag[s] = f ;
		}
		T4_SYNC() ;
	}
	if ( !useFlags )
	{
		if ( cx.tid == 0 )
			for ( int s = 0 ; s < st->nSeqs ; ++s )
				if ( t4_seq( cx, s )->consOff != 0 && !( t4_seq( cx, s )->flags & T4_CF_NOINDEX ) )
					s_update_consensus( cx, s, true ) ;
		T4_SYNC() ;
		return ;
	}
	for ( int s = 0 ; s < st->nSeqs ; ++s )
	{
		if ( !flag[s] )
			continue ;
		// UpdateConsensus( s, true ): drop the contig's k-mers, apply the changes, index it again
		T4Contig *seq = t4_seq( cx, s ) ;
		char *cons = t4_cons( cx, seq ) ;
		int *pw = t4_pw( cx, seq ) ;
		c_index_op( cx, cons, seq->len, T4_IDX_REMOVE, s, seq->barcode, 0, 0 ) ;
		T4_PAR_FOR( i, seq->len )
		{
			int max = 0, maxTag = 0 ;
			for ( int j = 0 ; j < 4 ; ++j )
				if ( pw[4 * i + j] > max )
				{
					max = pw[4 * i + j] ;
					maxTag = j ;
				}
			if ( max == 0 )
				continue ;
			int cur = t4_nuc( cons[i] ) ;
			if ( cur != maxTag && pw[4 * i + cur] < max )
				cons[i] = t4_numToNuc( maxTag ) ;
		}
		T4_SYNC() ;
		c_index_op( cx, cons, seq->len, T4_IDX_BUILD, s, seq->barcode, 0, 0 ) ;
	}
	T4_SYNC() ;
}

// SeqSet::IsContigShallow (SeqSet.hpp:2512-2556) on the uncompressed posWeight columns (the engine never compresses
// them; for a purged contig with flat coverage every column sums to numRead, which is the reference's
// `posWeight.Size() == 0` branch).  Serial.
T4_D inline int s_contig_shallow( T4Ctx &cx, int idx, int minCov )
{
	T4Contig *c = t4_seq( cx, idx ) ;
	if ( c->consOff == 0 )
		return 0 ;
	const int *pw = t4_pw( cx, c ) ;
	const int len = c->len ;
	int j ;
	for ( j = 0 ; j < len ; ++j )
		if ( pw[4 * j] + pw[4 * j + 1] + pw[4 * j + 2] + pw[4 * j + 3] >= minCov )
			break ;
	int start = j ;
	for ( j = len - 1 ; j >= start ; --j )
		if ( pw[4 * j] + pw[4 * j + 1] + pw[4 * j + 2] + pw[4 * j + 3] >= minCov )
			break ;
	int end = j ;
	for ( j = start ; j <= end ; ++j )
		if ( pw[4 * j] + pw[4 * j + 1] + pw[4 * j + 2] + pw[4 * j + 3] < minCov )
			break ;
	return ( j <= end || end < start ) ? 1 : 0 ;
}

// SeqSet::ReleaseFinishedBarcodeSeq( {barcode}, removeFromIndex = true, contigMinCov, earlyStop = true )
// (SeqSet.hpp:10815-10924), the only way the stage-1 driver calls it (main.cpp:1855).  Walks the slots from the end
// while they belong to `barcode` and are not purged yet: shallow contigs are dropped (index entries removed,
// ReleaseSeq), the others leave the index, get a final UpdateConsensus( i, false ) and, when their coverage is flat,
// numRead = that coverage.  The reference then compresses / frees posWeight -- storage only: Output prints the same
// numbers either way (SeqSet.hpp:10956-10992), so the columns stay as they are here.
T4_D T4_BIG void c_release_barcode( T4Ctx &cx, int barcode, int contigMinCov )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	T4_SYNC() ;
	for ( int i = st->nSeqs - 1 ; i >= 0 ; --i )
	{
		T4Contig *c = t4_seq( cx, i ) ;
		T4_SYNC() ;
		const bool dead = c->consOff == 0 ;
		const bool stop = !dead && ( ( c->flags & T4_CF_NOINDEX ) || c->barcode != barcode ) ;
		T4_SYNC() ;
		if ( dead )
			continue ;
		if ( stop )
			break ;
		int shallow = 0 ;
		if ( contigMinCov > 0 )
		{
			if ( cx.tid == 0 )
				sm->bi[0] = s_contig_shallow( cx, i, contigMinCov ) ;
			T4_SYNC() ;
			shallow = sm->bi[0] ;
			T4_SYNC() ;
		}
		c_index_op( cx, t4_cons( cx, c ), c->len, T4_IDX_REMOVE, i, c->barcode, 0, 0 ) ;
		if ( cx.tid == 0 )
		{
			if ( shallow )
				c->consOff = 0 ; // ReleaseSeq: the slot stays, Size() still counts it
			else
			{
				c->flags |= T4_CF_NOINDEX ;
				s_update_consensus( cx, i, false ) ;
				const char *cons = t4_cons( cx, c ) ;
				const int *pw = t4_pw( cx, c ) ;
				int cov = 0, j, k ;
				for ( j = 0 ; j < c->len ; ++j )
				{
					for ( k = 0 ; k < 4 ; ++k )
					{
						if ( k == t4_nuc( cons[j] ) )
						{
							if ( pw[4 * j + k] == 0 )
								break ;
							if ( j == 0 )
								cov = pw[4 * j + k] ;
							else if ( pw[4 * j + k] != cov )
								break ;
						}
						else if ( pw[4 * j + k] != 0 )
							break ;
					}
					if ( k < 4 )
						break ;
				}
				if ( j >= c->len )
					c->numRead = cov ;
			}
		}
		T4_SYNC() ;
	}
	T4_SYNC() ;
}

// SeqSet::ReleaseShallowContigs (SeqSet.hpp:10928): ReleaseSeq on every shallow contig; like the reference it leaves
// their index entries behind (the driver calls it after the last AddRead, main.cpp:1952-1955).
T4_D inline void c_release_shallow( T4Ctx &cx, int minCov )
{
	T4Stream *st = cx.st ;
	T4_SYNC() ;
	T4_PAR_FOR( i, st->nSeqs )
		if ( s_contig_shallow( cx, i, minCov ) )
			t4_seq( cx, i )->consOff = 0 ;
	T4_SYNC() ;
}

// Per-barcode read counters of the driver loop (main.cpp:1572-1581 barcodeTotalReadCount / barcodeReadCount): an
// open-addressing table over the barcodes of this stream's records.
struct T4BcTable
{
	u64 *key ;   // barcode + 1, 0 = empty
	u32 *total, *done ;
	u32 cap ;
} ;

T4_D inline u32 t4_bc_slot( const T4BcTable &t, int barcode, bool claim )
{
	u64 key = (u64)(u32)barcode + 1 ;
	u32 s = (u32)( ( key * 0x9E3779B97F4A7C15ull ) >> 33 ) & ( t.cap - 1 ) ;
	while ( 1 )
	{
		u64 kk = t.key[s] ;
		if ( kk == key )
			return s ;
		if ( kk == 0 )
		{
			if ( !claim )
				return 0xffffffffu ;
			u64 old = t4_atomic_cas( &t.key[s], 0ull, key ) ;
			if ( old == 0 || old == key )
				return s ;
		}
		s = ( s + 1 ) & ( t.cap - 1 ) ;
	}
}

// SeqSet::Clean(false) + ChangeKmerLength (SeqSet.hpp:4591-4629): compact the slots, rebuild the index.
// nomatchGapLimit is computed on the host (pow/log) and passed in.
T4_D T4_BIG void c_change_kmer_length( T4Ctx &cx, int kl, int nomatchGapLimit )
{
	T4Stream *st = cx.st ;
	T4_SYNC() ;
	T4Dir *dir = cx.P<T4Dir>( st->dirOff ) ;
	T4_PAR_FOR( i, st->dirCap ) // seqIndex.Clear()
		dir[i].key = 0 ;
	if ( cx.tid == 0 )
	{
		st->kmerLength = kl ;
		st->nomatchGapLimit = nomatchGapLimit ;
		st->dirUsed = 0 ;
		int k = 0 ;
		for ( int i = 0 ; i < st->nSeqs ; ++i )
		{
			T4Contig *c = t4_seq( cx, i ) ;
			if ( c->consOff == 0 )
				continue ;
			if ( k != i )
				*t4_seq( cx, k ) = *c ;
			++k ;
		}
		t4_set_prev( st, -1, -1, -1, -1, 0 ) ;
		st->nSeqs = k ;
	}
	T4_SYNC() ;
	for ( int i = 0 ; i < st->nSeqs ; ++i )
	{
		T4Contig *d = t4_seq( cx, i ) ;
		if ( d->flags & T4_CF_NOINDEX ) // Clean(): `if (seqs[k].index)` (SeqSet.hpp:4616)
			continue ;
		c_index_op( cx, t4_cons( cx, d ), d->len, T4_IDX_BUILD, i, d->barcode, 0, 0 ) ;
	}
	T4_SYNC() ;
}

// SeqSet::ComputeNomatchGapLimit (SeqSet.hpp:2476) for the k values the driver can reach
// (k = 9, 11, 13, 15, 17; main.cpp:1874-1879).  Values computed with the reference's own expression on the
// host (see t4_api: nomatch_gap_limit()); the device only needs them when the loop changes k by itself.
T4_D inline int t4_nomatch_gap_limit_table( int kl, const int *table )
{
	return table[kl] ;
}

// ---------------------------------------------------------------------------
// SeqSet::InputNovelRead (SeqSet.hpp:3028-3073).  Serial; reads cx.sm->read.
// ---------------------------------------------------------------------------
T4_D inline int c_input_novel_read( T4Ctx &cx, const char *id, int idLen, int len, int strand, int barcode )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	T4_SYNC() ;
	if ( cx.tid == 0 )
	{
		int seqIdx = s_new_contig( cx, len ) ;
		if ( seqIdx >= 0 )
		{
			T4Contig *c = t4_seq( cx, seqIdx ) ;
			s_set_name( cx, c, id, idLen ) ;
			c->barcode = barcode ;
			c->numRead = 1 ;
		}
		sm->bi[0] = seqIdx ;
	}
	T4_SYNC() ;
	int seqIdx = sm->bi[0] ;
	T4_SYNC() ;
	if ( seqIdx < 0 || st->error )
		return T4_E_NOMEM ;
	T4Contig *c = t4_seq( cx, seqIdx ) ;
	char *cons = t4_cons( cx, c ) ;
	int *pw = t4_pw( cx, c ) ;
	unsigned char *eq = t4_eq( cx, c ) ;
	const char *src = ( strand == -1 ) ? sm->rc : sm->read ;
	T4_PAR_FOR( i, len )
	{
		char ch = src[i] ;
		cons[i] = ch ;
		int w0 = 0, w1 = 0, w2 = 0, w3 = 0 ;
		if ( ch != 'N' )
		{
			int x = t4_nuc( ch ) ;
			w0 = x == 0 ; w1 = x == 1 ; w2 = x == 2 ; w3 = x == 3 ;
		}
		t4_col_put( pw, eq, i, w0, w1, w2, w3 ) ;
	}
	T4_SYNC() ;
	c_index_op( cx, cons, len, T4_IDX_BUILD, seqIdx, barcode, 0, 0 ) ;
	if ( cx.tid == 0 )
		t4_set_prev( st, seqIdx, 0, len - 1, 0, strand ) ;
	T4_SYNC() ;
	return seqIdx ;
}

// SeqSet::RepeatAddRead (SeqSet.hpp:4477-4507).  Collective.
T4_D inline int c_repeat_add_read( T4Ctx &cx, int len )
{
	T4Stream *st = cx.st ;
	if ( st->prevSeqIdx < 0 )
		return st->prevSeqIdx ;
	const char *r = ( st->prevStrand == -1 ) ? cx.sm->rc : cx.sm->read ;
	T4Contig *seq = t4_seq( cx, st->prevSeqIdx ) ;
	int *pw = t4_pw( cx, seq ) ;
	unsigned char *eq = t4_eq( cx, seq ) ;
	for ( int i = st->prevReadStart + cx.tid ; i <= st->prevReadEnd ; i += cx.nt )
	{
		if ( r[i] == 'N' )
			continue ;
		t4_col_add( pw, eq, i + st->prevSeqStart, t4_nuc( r[i] ), 1 ) ;
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
		++seq->numRead ;
	T4_SYNC() ;
	return st->prevSeqIdx ;
}

// L consecutive RepeatAddRead calls of the same read in one pass: the call only increments counters (SeqSet.hpp:4495-4501),
// so L calls add L.  The driver loop uses it for runs of duplicate records (c_run_loop).
T4_D inline int c_repeat_add_read_n( T4Ctx &cx, int len, int L )
{
	T4Stream *st = cx.st ;
	if ( st->prevSeqIdx < 0 )
		return st->prevSeqIdx ;
	const char *r = ( st->prevStrand == -1 ) ? cx.sm->rc : cx.sm->read ;
	T4Contig *seq = t4_seq( cx, st->prevSeqIdx ) ;
	int *pw = t4_pw( cx, seq ) ;
	unsigned char *eq = t4_eq( cx, seq ) ;
	for ( int i = st->prevReadStart + cx.tid ; i <= st->prevReadEnd ; i += cx.nt )
	{
		if ( r[i] == 'N' )
			continue ;
		t4_col_add( pw, eq, i + st->prevSeqStart, t4_nuc( r[i] ), L ) ;
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
		seq->numRead += L ;
	T4_SYNC() ;
	return st->prevSeqIdx ;
}

// Number of consecutive records from i on that carry T4_RD_DUP (record i included), at most cap.  Collective.
T4_D inline int c_dup_run_len( T4Ctx &cx, const t4_read_desc *descs, int i, int n, int cap )
{
	T4Smem *sm = cx.sm ;
	const int lim = ( n - i < cap ) ? n - i : cap ;
	T4_SYNC() ;
	if ( cx.tid == 0 )
		sm->bi[0] = lim ;
	T4_SYNC() ;
	for ( int base = 0 ; base < lim ; base += cx.nt )
	{
		const int t = base + cx.tid ;
		if ( t < lim && !( descs[i + t].flags & T4_RD_DUP ) )
		{
#if T4_CUDA
			atomicMin( &sm->bi[0], t ) ;
#else
			if ( t < sm->bi[0] )
				sm->bi[0] = t ;
#endif
		}
		T4_SYNC() ;
		const int v = sm->bi[0] ;
		T4_SYNC() ;
		if ( v < base + cx.nt )
			break ;
	}
	const int r = sm->bi[0] ;
	T4_SYNC() ;
	return r ;
}

// exact ExtendOverlap of overlap i on demand (thread 0 of the decision loop)
T4_D inline void s_make_exact( T4Ctx &cx, const char *r, int len, double factor, const T4Ovl *overlaps, T4Ovl *pre, int i )
{
#if T4_CUDA
	long long t0 = clock64() ;
#endif
	T4DpScratch ds = t4_dp_scratch( cx ) ;
	const u32 *bits = cx.P<u32>( cx.st->bitsOff ) ;
	T4Ovl e ;
	int ok = t4_extend_overlap( cx, r, len, t4_seq( cx, overlaps[i].seqIdx ), factor, ds, overlaps[i], e, bits + 32 * i, bits + 32 * i + 16 ) ;
	e.infoFromHits = ok ;
	e.hcCnt = 2 ;
	pre[i] = e ;
	t4_count( cx, 21, 1 ) ;
#if T4_CUDA
	t4_count( cx, 22, (u64)( clock64() - t0 ) ) ;
#endif
}

// Overhang side x = 2 i + right of overlap o = overlaps[i]: its posWeight columns *tw, their equality bytes *te and
// read bases *p.  Returns its length.
T4_D inline int t4_side_span( T4Ctx &cx, const T4Ovl &o, int right, const char *r, int len, const int **tw,
	const unsigned char **te, const char **p )
{
	T4Contig *seq = t4_seq( cx, o.seqIdx ) ;
	const T4Side s = t4_overhang_side( o, right, len, seq->len ) ;
	*tw = t4_pw( cx, seq ) + 4 * s.col ;
	*te = t4_eq( cx, seq ) + s.col ;
	*p = r + s.rp ;
	return s.n ;
}

// ExtendOverlap's overhang alignments of the sides pend[0 .. cnt) (each needs the banded DP): their statistics into
// sstats[side].  Collective.  On the device each warp takes two sides at a time, one per half-warp (w_side_pair);
// a side of 16 * T4_WACT_WORDS columns or more keeps its traceback and edit string in the arena scratch of its
// half-warp's first thread instead of shared memory.  The emulation aligns them one at a time.
T4_D inline void c_overhang_dps( T4Ctx &cx, const T4Ovl *overlaps, const char *r, int len, const u32 *bits, const int *pend, int cnt,
	T4SideStats *sstats )
{
#if T4_CUDA
	T4Smem *sm = cx.sm ;
	const int warp = cx.tid >> 5, nwarps = cx.nt >> 5, lane = cx.tid & 31 ;
	(void)bits ;
	for ( int q = 2 * warp ; q < cnt ; q += 2 * nwarps )
	{
		T4DpSide s[2] ;
#pragma unroll
		for ( int h = 0 ; h < 2 ; ++h )
		{
			T4DpSide &d = s[h] ;
			const int x = ( q + h < cnt ) ? pend[q + h] : -1 ;
			const int *tw = 0 ;
			d.te = 0 ;
			d.p = 0 ;
			d.n = ( x >= 0 ) ? t4_side_span( cx, overlaps[x >> 1], x & 1, r, len, &tw, &d.te, &d.p ) : 0 ;
			d.fromEnd = !( x & 1 ) ;
			const bool small = d.n < 16 * T4_WACT_WORDS ;
			d.act = small ? sm->wact[warp][h] : (u32 *)t4_dp_scratch_of( cx, warp * 32 + 16 * h ).act ;
			d.actStride = small ? T4_WACT_WORDS : (int)( T4_DP_STRIDE / 4 ) ;
			d.al = small ? sm->wal[warp][h] : t4_align_of_thread( cx, warp * 32 + 16 * h ) ;
			d.alCap = small ? (int)sizeof( sm->wal[0][0] ) : 2 * T4_DEV_MAX_READ + 8 ;
		}
		T4SideStats r0, r1 ;
		w_side_pair( cx, s[0], s[1], sm->wnib[warp], sm->wbits[warp], r0, r1 ) ;
		if ( lane == 0 )
		{
			sstats[pend[q]] = r0 ;
			if ( q + 1 < cnt )
				sstats[pend[q + 1]] = r1 ;
			t4_count( cx, 1, ( q + 1 < cnt ) ? 2 : 1 ) ;
		}
	}
#else
	T4DpScratch ds = t4_dp_scratch( cx ) ;
	T4_PAR_FOR( q, cnt )
	{
		const int x = pend[q] ;
		const int *tw ;
		const unsigned char *te ;
		const char *p ;
		const int n = t4_side_span( cx, overlaps[x >> 1], x & 1, r, len, &tw, &te, &p ) ;
		(void)te ;
		T4AlignView av = t4_overhang_align( tw, p, n, bits + 32 * ( x >> 1 ) + 16 * ( x & 1 ), ds ) ;
		if ( av.dp )
			t4_count( cx, 1, 1 ) ;
		sstats[x] = t4_side_stats( av, !( x & 1 ) ) ;
	}
#endif
	T4_SYNC() ;
}

// IsBaseEqual( column, read base ) from the column's equality byte (t4_eq): an 'N' read base matches every column.
T4_HD inline bool t4_eq_hit( unsigned b, char pc ) { return pc == 'N' || ( ( b >> t4_nuc( pc ) ) & 1u ) ; }

// A side of n overhang columns with `matches` diagonal matches needs the banded DP (AlignAlgo.hpp:59-103: more than
// 2 mismatches on the diagonal).
T4_HD inline bool t4_side_needs_dp( int n, int matches )
{
	return n >= 2 && ( SCORE_MATCH * matches + SCORE_MISMATCH * ( n - matches ) < n * SCORE_MATCH + 2 * SCORE_INDEL ) ;
}

#if T4_CUDA
// The overhang masks of overlap o for one warp (ExtendOverlap, SeqSet.hpp:1165-1175): bit t of word w of a side is
// IsBaseEqual( column, read base ) of overhang position 32 w + t.  Lane w < 16 returns word w of the left side, lane
// 16 + w word w of the right side (the layout of st->bitsOff), zero beyond the side; *nL / *nR get the side lengths.
// The equality bytes of both sides are loaded 8 words at a time (one round trip for overhangs up to 256 columns)
// before any of them is used.
T4_D inline u32 w_overhang_masks( T4Ctx &cx, const T4Ovl &o, const char *r, int len, int lane, int *nL, int *nR )
{
	T4Contig *seq = t4_seq( cx, o.seqIdx ) ;
	const unsigned char *eq = t4_eq( cx, seq ) ;
	const T4Side sL = t4_overhang_side( o, 0, len, seq->len ), sR = t4_overhang_side( o, 1, len, seq->len ) ;
	const int L = sL.n, R = sR.n ;
	const unsigned char *eL = eq + sL.col, *eR = eq + sR.col ;
	const char *pL = r + sL.rp, *pR = r + sR.rp ;
	const int nw = ( t4_max( L, R ) + 31 ) >> 5 ;
	u32 mine = 0 ;
	for ( int w0 = 0 ; w0 < nw ; w0 += 8 )
	{
		unsigned bl[8], br[8] ;
#pragma unroll
		for ( int u = 0 ; u < 8 ; ++u )
		{
			const int t = 32 * ( w0 + u ) + lane ;
			bl[u] = t < L ? eL[t] : 0u ;
			br[u] = t < R ? eR[t] : 0u ;
		}
#pragma unroll
		for ( int u = 0 ; u < 8 ; ++u )
		{
			const int t = 32 * ( w0 + u ) + lane ;
			const u32 ml = __ballot_sync( T4_FULL, t < L && t4_eq_hit( bl[u], pL[t] ) ) ;
			const u32 mr = __ballot_sync( T4_FULL, t < R && t4_eq_hit( br[u], pR[t] ) ) ;
			if ( lane == w0 + u )
				mine = ml ;
			if ( lane == 16 + w0 + u )
				mine = mr ;
		}
	}
	*nL = L ;
	*nR = R ;
	return mine ;
}
#endif

// IsBaseEqual( column, read base ) of every overhang column of every overlap (ExtendOverlap, SeqSet.hpp:1165-1175) as bit
// masks: bits[32 * i + 16 * side + w] holds overhang positions 32 w .. 32 w + 31 of side (0 left, 1 right) of overlap i.
// Collective; r is the read in the strand of the overlaps.  The emulation's form of w_overhang_masks.
#if !T4_CUDA
T4_D inline void c_overhang_bits( T4Ctx &cx, const T4Ovl *overlaps, int overlapCnt, const char *r, int len, u32 *bits )
{
	T4_PAR_FOR( x, overlapCnt * 32 )
	{
		int oi = x >> 5, w = x & 15, right = ( x >> 4 ) & 1 ;
		const T4Ovl &o = overlaps[oi] ;
		T4Contig *seq = t4_seq( cx, o.seqIdx ) ;
		const T4Side s = t4_overhang_side( o, right, len, seq->len ) ;
		u32 m = 0 ;
		if ( w * 32 < s.n )
		{
			const unsigned char *eq = t4_eq( cx, seq ) ;
			int hi = s.n - w * 32 < 32 ? s.n - w * 32 : 32 ;
			for ( int t = 0 ; t < hi ; ++t )
				if ( t4_eq_hit( eq[s.col + w * 32 + t], r[s.rp + w * 32 + t] ) )
					m |= 1u << t ;
		}
		bits[x] = m ;
	}
	T4_SYNC() ;
}
#endif

// Lazy ExtendOverlap: pre[i] of c_add_read from the statistics of overlap i's two sides (ind == -1: deferred to the
// banded DP).  With both sides settled it is the exact result (state 2: hcCnt 2, infoFromHits = the return value).
// Otherwise, when the return value alone matters (the bridging loop, SeqSet.hpp:3736-3750), an overlap is skipped
// without any DP if ExtendOverlap provably returns 0 (state 1): with the total diagonal mismatch count M over the
// mismatch budget and density, either every deferred side aligns without indel (then its counts ARE the diagonal
// counts and the budget test fails) or some side has an indel (ret = 0).  State 0 leaves it to the DP pass.
T4_D inline T4Ovl t4_settle_overlap( T4Ctx &cx, int len, T4Contig *seq, double factor, const T4Ovl &o, const T4SideStats &ls,
	const T4SideStats &rs )
{
	T4Ovl e = o ;
	if ( ls.ind == 0 && rs.ind == 0 )
	{
		int ok = t4_extend_finish( cx, len, seq, factor, o, e, ls, rs ) ;
		e.infoFromHits = ok ; // aux: the return value
		e.hcCnt = 2 ;         // aux: exact
	}
	else
	{
		int L = t4_overhang_side( o, 0, len, seq->len ).n ;
		int R = t4_overhang_side( o, 1, len, seq->len ).n ;
		int M = ls.x + rs.x ;
		int thr = 2 + ( L >= 2 ? 1 : 0 ) + ( R >= 2 ? 1 : 0 ) ;
		thr = (int)( thr * factor ) ;
		bool surely0 = ( M > thr ) && ( (double)M / ( L + R ) > 1.5 / cx.st->kmerLength ) ;
		e.infoFromHits = 0 ;
		e.hcCnt = surely0 ? 1 : 0 ;
	}
	return e ;
}

// ExtendOverlap's overhang masks and side statistics of every overlap, and pre[i] (t4_settle_overlap); the sides that
// need the DP get ind == -1 in sstats[2 i + side].  The masks also go to bits (the DPs of the emulation and
// s_make_exact read them).  Collective.  On the device one warp takes an overlap at a time: record and contig header
// once, the equality bytes of both sides in one batch, the masks in registers (and the warp's shared words for the
// statistics), then lane 0 settles the overlap -- no CTA barrier between masks and results.
T4_D inline void c_overhang_settle( T4Ctx &cx, const T4Ovl *overlaps, int overlapCnt, const char *r, int len, double factor,
	u32 *bits, T4SideStats *sstats, T4Ovl *pre )
{
#if T4_CUDA
	const int warp = cx.tid >> 5, nwarps = cx.nt >> 5, lane = cx.tid & 31 ;
	u32 *wb = &cx.sm->wbits[warp][0][0] ; // [side][word], the layout of one overlap's 32 words of bits
	for ( int oi = warp ; oi < overlapCnt ; oi += nwarps )
	{
		const T4Ovl o = overlaps[oi] ;
		int n[2] ;
		const u32 mine = w_overhang_masks( cx, o, r, len, lane, &n[0], &n[1] ) ;
		bits[32 * oi + lane] = mine ;
		wb[lane] = mine ;
		int mc = __popc( mine ) ;
		mc += __shfl_xor_sync( T4_FULL, mc, 8 ) ;
		mc += __shfl_xor_sync( T4_FULL, mc, 4 ) ;
		mc += __shfl_xor_sync( T4_FULL, mc, 2 ) ;
		mc += __shfl_xor_sync( T4_FULL, mc, 1 ) ;
		const int matches[2] = { __shfl_sync( T4_FULL, mc, 0 ), __shfl_sync( T4_FULL, mc, 16 ) } ;
		__syncwarp() ;
		T4SideStats ss[2] ;
#pragma unroll
		for ( int right = 0 ; right < 2 ; ++right )
		{
			if ( !t4_side_needs_dp( n[right], matches[right] ) )
			{
				T4AlignView av ;
				av.a = 0 ; av.bits = wb + 16 * right ; av.n = n[right] ; av.dp = 0 ;
				ss[right] = w_side_stats( av, !right, lane ) ;
			}
			else
			{
				ss[right].m = matches[right] ;
				ss[right].x = n[right] - matches[right] ;
				ss[right].ind = -1 ; // deferred
				ss[right].good = 0 ;
			}
		}
		if ( lane == 0 )
		{
			sstats[2 * oi] = ss[0] ;
			sstats[2 * oi + 1] = ss[1] ;
			pre[oi] = t4_settle_overlap( cx, len, t4_seq( cx, o.seqIdx ), factor, o, ss[0], ss[1] ) ;
		}
		__syncwarp() ;
	}
#else
	c_overhang_bits( cx, overlaps, overlapCnt, r, len, bits ) ;
	T4_PAR_FOR( i, overlapCnt )
	{
		const T4Ovl &o = overlaps[i] ;
		T4Contig *seq = t4_seq( cx, o.seqIdx ) ;
		T4SideStats ss[2] ;
		for ( int right = 0 ; right < 2 ; ++right )
		{
			int n = t4_overhang_side( o, right, len, seq->len ).n ;
			const u32 *bb = bits + 32 * i + 16 * right ;
			int matches = 0 ;
			for ( int w = 0 ; w * 32 < n ; ++w )
				matches += __builtin_popcount( bb[w] ) ;
			if ( !t4_side_needs_dp( n, matches ) )
			{
				T4AlignView av ;
				av.a = 0 ; av.bits = bb ; av.n = n ; av.dp = 0 ;
				ss[right] = t4_side_stats( av, !right ) ;
			}
			else
			{
				ss[right].m = matches ;
				ss[right].x = n - matches ;
				ss[right].ind = -1 ; // deferred
				ss[right].good = 0 ;
			}
			sstats[2 * i + right] = ss[right] ;
		}
		pre[i] = t4_settle_overlap( cx, len, seq, factor, o, ss[0], ss[1] ) ;
	}
#endif
	T4_SYNC() ;
}

// ---------------------------------------------------------------------------
// ExtendOverlap of every overlap of a read: the one pass of AddRead and AssignRead
// ---------------------------------------------------------------------------

// ExtendOverlap (SeqSet.hpp:1165-1277) of every overlap into pre[i]: hcCnt 2 (exact) and infoFromHits = the return
// value, or one of t4_settle_overlap's lazy states.  Collective; r is the read in the strand of the overlaps.  The
// masks and side statistics of every overlap come from c_overhang_settle; the sides that need the banded DP are then
// aligned in one parallel pass (c_overhang_dps), all of them except, when the read is easy, those of a provably-0
// overlap (state 1).  A read is easy when pre[0] is exact, extends, covers the whole read and is at least
// easySimilarity similar: a caller that then consults the other overlaps only through their return value may leave
// them so.  No similarity exceeds 1, so an easySimilarity above 1 makes every overlap exact.
// Borrows st->failOff for the side statistics and the list of sides to align; the masks stay in st->bitsOff, where
// s_make_exact reads them.  Returns whether the read is easy.  clk (may be 0): thread 0's clock64() after the settle
// pass and after the list (device only).
T4_D inline bool c_extend_overlaps( T4Ctx &cx, const T4Ovl *overlaps, int overlapCnt, const char *r, int len, double factor,
	double easySimilarity, T4Ovl *pre, long long *clk )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	if ( cx.tid == 0 )
		t4_count( cx, 16, (u64)overlapCnt ) ;
	u32 *bits = cx.P<u32>( st->bitsOff ) ;
	T4SideStats *sstats = (T4SideStats *)cx.P<char>( st->failOff ) ; // 2 per overlap
	c_overhang_settle( cx, overlaps, overlapCnt, r, len, factor, bits, sstats, pre ) ;
#if T4_CUDA
	if ( clk && cx.tid == 0 )
		clk[0] = clock64() ;
#endif
	bool easy = ( pre[0].hcCnt == 2 && pre[0].infoFromHits == 1 && pre[0].similarity >= easySimilarity
		&& pre[0].readStart == 0 && pre[0].readEnd == len - 1 ) ;
	int *pend = (int *)( sstats + 2 * overlapCnt ) ; // the sides to align, in side order (failOff holds a T4Ovl per overlap)
#if T4_CUDA
	if ( cx.tid < 32 )
	{
		int cnt = 0 ;
		for ( int base = 0 ; base < 2 * overlapCnt ; base += 32 )
		{
			int x = base + cx.tid ;
			bool p = x < 2 * overlapCnt && sstats[x].ind == -1 && !( easy && pre[x >> 1].hcCnt == 1 ) ;
			unsigned m = __ballot_sync( T4_FULL, p ) ;
			if ( p )
				pend[cnt + __popc( m & ( ( 1u << cx.tid ) - 1u ) )] = x ;
			cnt += __popc( m ) ;
		}
		if ( cx.tid == 0 )
			sm->bi[0] = cnt ;
	}
#else
	{
		int cnt = 0 ;
		for ( int x = 0 ; x < 2 * overlapCnt ; ++x )
			if ( sstats[x].ind == -1 && !( easy && pre[x >> 1].hcCnt == 1 ) )
				pend[cnt++] = x ;
		sm->bi[0] = cnt ;
	}
#endif
	T4_SYNC() ;
#if T4_CUDA
	if ( clk && cx.tid == 0 )
		clk[1] = clock64() ;
#endif
	c_overhang_dps( cx, overlaps, r, len, bits, pend, sm->bi[0], sstats ) ;
	T4_PAR_FOR( i, overlapCnt )
	{
		if ( pre[i].hcCnt == 2 || sstats[2 * i].ind == -1 || sstats[2 * i + 1].ind == -1 )
			continue ;
		T4Ovl e ;
		int ok = t4_extend_finish( cx, len, t4_seq( cx, overlaps[i].seqIdx ), factor, overlaps[i], e, sstats[2 * i], sstats[2 * i + 1] ) ;
		e.infoFromHits = ok ;
		e.hcCnt = 2 ;
		pre[i] = e ;
	}
	T4_SYNC() ;
	return easy ;
}

// ---------------------------------------------------------------------------
// SeqSet::AddRead (SeqSet.hpp:3426-4473), novel-contig set, in its phases.  c_add_read calls them in order; the
// decision and the merge hand the collective phases their result in cx.sm->plan.
// ---------------------------------------------------------------------------

// Gene-name prefix filter (SeqSet.hpp:3445-3472): keeps, in order, the overlaps whose contig name does not start with
// a capital letter, starts with the first three letters of geneName, or is "Novel".  Collective; the walk is thread
// 0's.  Returns the new overlap count.
T4_D inline int c_gene_filter( T4Ctx &cx, T4Ovl *overlaps, int overlapCnt, const char *geneName )
{
	T4Smem *sm = cx.sm ;
	if ( cx.tid == 0 )
	{
		int k = 0 ;
		for ( int i = 0 ; i < overlapCnt ; ++i )
		{
			T4Contig *c = t4_seq( cx, overlaps[i].seqIdx ) ;
			const char *nm = cx.P<char>( c->nameOff ) ;
			int j = 3 ;
			if ( nm[0] >= 'A' && nm[0] <= 'Z' )
			{
				for ( j = 0 ; j < 3 ; ++j )
					if ( nm[j] != geneName[j] )
						break ;
			}
			if ( j == 3 || t4_name_eq( nm, c->nameLen, "Novel", 5 ) )
			{
				if ( k != i )
					overlaps[k] = overlaps[i] ;
				++k ;
			}
		}
		sm->bi[0] = k ;
	}
	T4_SYNC() ;
	overlapCnt = sm->bi[0] ;
	T4_SYNC() ;
	return overlapCnt ;
}

// The decision walk (SeqSet.hpp:3476-3877): from the sorted overlaps and their ExtendOverlap results pre[] to the
// extended overlaps to commit, extendedOverlaps[0 .. k), updating the contigs' extension anchors on the way.  Makes an
// overlap exact on demand (s_make_exact) where pre[] holds no exact result.  Thread 0.  Borrows st->failOff for the
// failed extended overlaps and st->anchorOff for the old anchors.  Returns k; sortExtendedOverlaps: whether the merge
// sorts the extended overlaps by read start.
T4_D inline int s_decide_overlaps( T4Ctx &cx, const T4Ovl *overlaps, int overlapCnt, const char *r, int len, double factor, T4Ovl *pre,
	int minKmerCount, double similarityThreshold, T4Ovl *extendedOverlaps, bool &sortExtendedOverlaps )
{
	T4Stream *st = cx.st ;
	T4Ovl *failedExtendedOverlaps = cx.P<T4Ovl>( st->failOff ) ;
	int *oldMinExtAnchor = cx.P<int>( st->anchorOff ) ;
	const int radius = st->radius ;
	int i, j, k = 0 ;
	int failedExtendedOverlapsCnt = 0 ;
	T4Ovl goodExtendedOverlap ;
	goodExtendedOverlap.seqIdx = -1 ;
	int tag = 0 ;
	sortExtendedOverlaps = true ;

	for ( i = 0 ; i < overlapCnt ; ++i )
	{
		T4Contig *seq = t4_seq( cx, overlaps[i].seqIdx ) ;
		oldMinExtAnchor[2 * i] = seq->minLeftExtAnchor ;
		oldMinExtAnchor[2 * i + 1] = seq->minRightExtAnchor ;
		for ( j = 0 ; j < k ; ++j )
		{
			int leftRadius = radius, rightRadius = radius ;
			if ( extendedOverlaps[j].seqStart == 0 )
				leftRadius = 0 ;
			if ( extendedOverlaps[j].seqEnd == t4_seq( cx, extendedOverlaps[j].seqIdx )->len - 1 )
				rightRadius = 0 ;
			if ( overlaps[i].readStart >= extendedOverlaps[j].readStart - leftRadius
				&& overlaps[i].readEnd <= extendedOverlaps[j].readEnd + rightRadius
				&& ( overlaps[i].seqStart >= radius || overlaps[i].seqEnd <= seq->len - radius - 1 ) )
				break ;
			leftRadius = radius ;
			rightRadius = radius ;
			if ( overlaps[i].seqStart == 0 )
				leftRadius = 0 ;
			if ( overlaps[i].seqEnd == seq->len - 1 )
				rightRadius = 0 ;
			if ( extendedOverlaps[j].readStart >= overlaps[i].readStart - leftRadius
				&& extendedOverlaps[j].readEnd <= overlaps[i].readEnd + rightRadius )
				break ;
		}
		if ( j < k )
			continue ;
		if ( pre[i].hcCnt != 2 )
			s_make_exact( cx, r, len, factor, overlaps, pre, i ) ;
		extendedOverlaps[k] = pre[i] ;
		if ( pre[i].infoFromHits == 1 )
		{
			T4Ovl &eo = extendedOverlaps[k] ;
			if ( eo.similarity < similarityThreshold )
			{
				if ( ( minKmerCount <= 1 || eo.similarity + 0.01 >= similarityThreshold ) && eo.readStart == 0
					&& eo.readEnd == len - 1 )
					goodExtendedOverlap = eo ;
				continue ;
			}
			for ( j = 0 ; j < k ; ++j )
			{
				int leftRadius = radius, rightRadius = radius ;
				if ( extendedOverlaps[j].seqStart == 0 )
					leftRadius = 0 ;
				if ( extendedOverlaps[j].seqEnd == t4_seq( cx, extendedOverlaps[j].seqIdx )->len - 1 )
					rightRadius = 0 ;
				if ( eo.readStart >= extendedOverlaps[j].readStart - leftRadius
					&& eo.readEnd <= extendedOverlaps[j].readEnd + rightRadius
					&& ( overlaps[i].seqStart > 0 || overlaps[i].seqEnd < seq->len - 1 ) )
					break ;
				if ( extendedOverlaps[j].readStart >= eo.readStart - radius && extendedOverlaps[j].readEnd <= eo.readEnd + radius )
					break ;
			}
			if ( j < k )
				continue ;
			T4Contig *eseq = t4_seq( cx, eo.seqIdx ) ;
			int span = eo.readEnd - eo.readStart + 1 ;
			for ( j = 0 ; j < i ; ++j )
			{
				if ( eo.seqStart == 0 && eo.seqEnd == eseq->len - 1 )
					continue ;
				if ( eo.readStart >= overlaps[j].readStart && eo.readEnd <= overlaps[j].readEnd
					&& ( overlaps[j].readEnd - overlaps[j].readStart >= eo.readEnd - eo.readStart + 10
						|| overlaps[j].similarity + 0.02 >= eo.similarity ) )
				{
					if ( eo.readStart > 0 && eseq->minLeftExtAnchor < span )
						eseq->minLeftExtAnchor = span ;
					if ( eo.readEnd < len - 1 && eseq->minRightExtAnchor < span )
						eseq->minRightExtAnchor = span ;
					break ;
				}
			}
			if ( j < i )
				continue ;
			for ( j = 0 ; j < failedExtendedOverlapsCnt ; ++j )
			{
				if ( eo.seqStart == 0 && eo.seqEnd == eseq->len - 1 )
					continue ;
				if ( eo.readStart >= failedExtendedOverlaps[j].readStart && eo.readEnd <= failedExtendedOverlaps[j].readEnd )
				{
					if ( eo.readStart > 0 && eseq->minLeftExtAnchor < span )
						eseq->minLeftExtAnchor = span ;
					if ( eo.readEnd < len - 1 && eseq->minRightExtAnchor < span )
						eseq->minRightExtAnchor = span ;
					break ;
				}
			}
			if ( j < failedExtendedOverlapsCnt )
				continue ;
			if ( eo.readStart > 0 && eseq->minLeftExtAnchor >= span )
				continue ;
			if ( eo.readEnd < len - 1 && eseq->minRightExtAnchor >= span )
				continue ;
			tag = i ;
			++k ;
		}
		else
		{
			failedExtendedOverlaps[failedExtendedOverlapsCnt] = extendedOverlaps[k] ;
			++failedExtendedOverlapsCnt ;
		}
	}

	if ( k == 1 && extendedOverlaps[0].readStart <= radius && extendedOverlaps[0].readEnd >= len - radius )
	{
		// could the read bridge to a second contig? (SeqSet.hpp:3732-3793)
		for ( i = 0 ; i < overlapCnt ; ++i )
		{
			if ( tag == i )
				continue ;
			if ( pre[i].hcCnt == 1 )
				continue ; // ExtendOverlap provably returns 0; only the return value is consulted here
			if ( pre[i].hcCnt != 2 )
				s_make_exact( cx, r, len, factor, overlaps, pre, i ) ;
			extendedOverlaps[k] = pre[i] ;
			if ( pre[i].infoFromHits == 1 )
			{
				j = i ;
				++k ;
			}
		}
		if ( k > 2 )
			k = 1 ;
		else if ( k == 2 )
		{
			int span = extendedOverlaps[1].readEnd - extendedOverlaps[1].readStart + 1 ;
			if ( extendedOverlaps[1].readStart > 0 && oldMinExtAnchor[2 * j] >= span )
				k = 1 ;
			if ( extendedOverlaps[1].readEnd < len - 1 && oldMinExtAnchor[2 * j + 1] >= span )
				k = 1 ;
			if ( k == 2 )
			{
				if ( extendedOverlaps[0].seqEnd == t4_seq( cx, extendedOverlaps[0].seqIdx )->len - 1
					&& extendedOverlaps[1].seqStart == 0 )
					sortExtendedOverlaps = false ;
				else if ( extendedOverlaps[0].seqStart == 0
					&& extendedOverlaps[1].seqEnd == t4_seq( cx, extendedOverlaps[1].seqIdx )->len - 1 )
				{
					sortExtendedOverlaps = false ;
					T4Ovl tmp = extendedOverlaps[0] ;
					extendedOverlaps[0] = extendedOverlaps[1] ;
					extendedOverlaps[1] = tmp ;
				}
				else
					k = 1 ;
			}
		}
	}

	if ( similarityThreshold > st->novelSeqSimilarity )
	{
		int cnt = 0 ;
		for ( i = 0 ; i < k ; ++i )
			if ( extendedOverlaps[i].similarity >= similarityThreshold )
			{
				extendedOverlaps[cnt] = extendedOverlaps[i] ;
				++cnt ;
			}
		k = cnt ;
	}
	if ( k == 0 && goodExtendedOverlap.seqIdx != -1 )
	{
		extendedOverlaps[0] = goodExtendedOverlap ;
		k = 1 ;
	}
	if ( k > 1 )
	{
		for ( i = 0 ; i < k ; ++i )
			if ( extendedOverlaps[i].similarity >= 0.95 )
				break ;
		if ( i >= k )
		{
			int maxtag = 0 ;
			for ( i = 1 ; i < k ; ++i )
				if ( t4_ovl_less( extendedOverlaps[i], extendedOverlaps[maxtag] ) )
					maxtag = i ;
			extendedOverlaps[0] = extendedOverlaps[maxtag] ;
			k = 1 ;
		}
	}
	if ( k > 1 )
	{
		for ( i = 0 ; i < k - 1 ; ++i )
			for ( j = i + 1 ; j < k ; ++j )
				if ( extendedOverlaps[i].seqIdx == extendedOverlaps[j].seqIdx )
				{
					k = 0 ;
					break ;
				}
	}
	return k ;
}

// The merge commit (SeqSet.hpp:3878-4130) of the k > 1 extended overlaps extendedOverlaps[0 .. k): one contig from all
// of them and the read.  Rare (0.7 % of AddReads).  Thread 0.  Writes plan's kind, added, bail, ret, seqIdx and
// readInConsensusOffset.  Borrows seqOffset (st->extOff, whose pre[] is dead after the decision) for the contigs'
// positions in the merged contig.
T4_D inline void s_merge_commit( T4Ctx &cx, T4Ovl *extendedOverlaps, int k, bool sortExtendedOverlaps, const char *r, int len,
	int barcode, int *seqOffset, T4AddPlan &plan )
{
	int i, j ;
	int eOverlapCnt = k ;
	plan.added = true ;
	plan.kind = 2 ;
	if ( sortExtendedOverlaps )
	{
		// std::sort by readStart only; equal keys would make the order implementation defined, so keep the
		// sort stable and flag ties (they need differing contigs with equal extended read starts)
		for ( i = 1 ; i < eOverlapCnt ; ++i )
		{
			T4Ovl x = extendedOverlaps[i] ;
			for ( j = i - 1 ; j >= 0 && extendedOverlaps[j].readStart > x.readStart ; --j )
				extendedOverlaps[j + 1] = extendedOverlaps[j] ;
			extendedOverlaps[j + 1] = x ;
		}
	}
	for ( i = 0 ; i < k && !plan.bail ; ++i )
		for ( j = i + 1 ; j < k ; ++j )
		{
			T4Contig *ca = t4_seq( cx, extendedOverlaps[i].seqIdx ) ;
			T4Contig *cb = t4_seq( cx, extendedOverlaps[j].seqIdx ) ;
			if ( !t4_name_compatible( cx.P<char>( ca->nameOff ), ca->nameLen, cx.P<char>( cb->nameOff ), cb->nameLen ) )
			{
				plan.bail = true ;
				break ;
			}
		}
	if ( plan.bail )
		plan.ret = -1 ;
	else
	{
		int sum = 0 ;
		for ( i = 0 ; i < eOverlapCnt ; ++i )
			sum += t4_seq( cx, extendedOverlaps[i].seqIdx )->len ;
		// positions of the contigs in the merged contig
		if ( extendedOverlaps[0].readStart > 0 )
		{
			for ( i = 0 ; i < eOverlapCnt ; ++i )
				seqOffset[i] = extendedOverlaps[i].readStart ;
		}
		else
		{
			seqOffset[0] = 0 ;
			for ( i = 1 ; i < eOverlapCnt ; ++i )
				seqOffset[i] = seqOffset[i - 1] + t4_seq( cx, extendedOverlaps[i - 1].seqIdx )->len - 1
					+ ( extendedOverlaps[i].readStart - extendedOverlaps[i - 1].readEnd ) ;
		}
		u64 ncOff = s_alloc( cx, (u64)( sum + len + 1 ) + 16 ) ;
		if ( ncOff )
		{
			char *newConsensus = cx.P<char>( ncOff ) ;
			if ( extendedOverlaps[0].readStart > 0 )
				memcpy( newConsensus, r, len ) ;
			else
				memcpy( newConsensus + extendedOverlaps[0].seqStart, r, len ) ;
			for ( i = eOverlapCnt - 1 ; i >= 0 ; --i )
			{
				T4Contig *c = t4_seq( cx, extendedOverlaps[i].seqIdx ) ;
				memcpy( newConsensus + seqOffset[i], t4_cons( cx, c ), c->len ) ;
			}
			int newConsensusLen = 0 ;
			int lastEndExtendedOverlapIdx = eOverlapCnt - 1 ;
			k = 0 ;
			for ( i = 0 ; i < eOverlapCnt ; ++i )
			{
				int e = seqOffset[i] + t4_seq( cx, extendedOverlaps[i].seqIdx )->len ;
				if ( e > k )
				{
					k = e ;
					lastEndExtendedOverlapIdx = i ;
				}
			}
			if ( extendedOverlaps[lastEndExtendedOverlapIdx].readEnd < len )
				newConsensusLen = k + ( len - extendedOverlaps[lastEndExtendedOverlapIdx].readEnd - 1 ) ;
			else
				newConsensusLen = k ;

			int newSeqIdx = extendedOverlaps[0].seqIdx ;
			k = 0 ;
			for ( i = 1 ; i < eOverlapCnt ; ++i )
				if ( extendedOverlaps[i].seqIdx < newSeqIdx )
				{
					newSeqIdx = extendedOverlaps[i].seqIdx ;
					k = i ;
				}
			// index removal uses the OLD consensus of every participant
			for ( i = 0 ; i < eOverlapCnt ; ++i )
			{
				T4Contig *c = t4_seq( cx, extendedOverlaps[i].seqIdx ) ;
				s_remove_index( cx, t4_cons( cx, c ), c->len, extendedOverlaps[i].seqIdx, barcode, 0 ) ;
			}
			// new posWeight: old columns of newSeqIdx shifted by seqOffset[k], zero elsewhere, plus the others
			T4Contig *ns = t4_seq( cx, newSeqIdx ) ;
			int oldLen = ns->len ;
			int cap = 2 * newConsensusLen + 128 ;
			u64 co = s_alloc( cx, cap ) ;
			u64 po = s_alloc( cx, T4_PW_BYTES( cap ) ) ;
			if ( co && po )
			{
				int lead = ( cap - newConsensusLen ) / 2 ;
				int *npw = cx.P<int>( po ) + 4 * lead ;
				unsigned char *neq = cx.P<unsigned char>( po + 16ull * cap ) + lead ;
				int *opw = t4_pw( cx, ns ) ;
				for ( i = 0 ; i < 4 * newConsensusLen ; ++i )
					npw[i] = 0 ;
				for ( i = 0 ; i < 4 * oldLen ; ++i )
					npw[4 * seqOffset[k] + i] = opw[i] ;
				for ( i = 0 ; i < eOverlapCnt ; ++i )
				{
					int sIdx = extendedOverlaps[i].seqIdx ;
					if ( sIdx == newSeqIdx )
						continue ;
					T4Contig *c = t4_seq( cx, sIdx ) ;
					ns->numRead += c->numRead ;
					int *cpw = t4_pw( cx, c ) ;
					for ( j = 0 ; j < 4 * c->len ; ++j )
						npw[4 * seqOffset[i] + j] += cpw[j] ;
				}
				for ( i = 0 ; i < newConsensusLen ; ++i )
					neq[i] = (unsigned char)t4_eq_nibble( npw + 4 * i ) ;
				// name (SeqSet.hpp:4066-4096)
				int nameIdx ;
				for ( nameIdx = 0 ; nameIdx < eOverlapCnt ; ++nameIdx )
				{
					T4Contig *c = t4_seq( cx, extendedOverlaps[nameIdx].seqIdx ) ;
					if ( !t4_name_eq( cx.P<char>( c->nameOff ), c->nameLen, "Novel", 5 ) )
						break ;
				}
				if ( nameIdx >= eOverlapCnt )
					nameIdx = 0 ;
				int nameSum = 0 ;
				for ( i = 0 ; i < eOverlapCnt ; ++i )
					nameSum += t4_seq( cx, extendedOverlaps[i].seqIdx )->nameLen ;
				u64 nbOff = s_alloc( cx, nameSum + eOverlapCnt + 1 ) ;
				if ( nbOff )
				{
					char *nameBuffer = cx.P<char>( nbOff ) ;
					T4Contig *c0 = t4_seq( cx, extendedOverlaps[nameIdx].seqIdx ) ;
					memcpy( nameBuffer, cx.P<char>( c0->nameOff ), c0->nameLen ) ;
					int nl = c0->nameLen ;
					for ( i = 0 ; i < eOverlapCnt ; ++i )
					{
						if ( i == nameIdx )
							continue ;
						if ( i > 0 )
						{
							T4Contig *ci = t4_seq( cx, extendedOverlaps[i].seqIdx ) ;
							T4Contig *cp = t4_seq( cx, extendedOverlaps[i - 1].seqIdx ) ;
							if ( !t4_name_eq( cx.P<char>( ci->nameOff ), ci->nameLen, cx.P<char>( cp->nameOff ), cp->nameLen ) )
							{
								nameBuffer[nl] = '+' ;
								memcpy( nameBuffer + nl + 1, cx.P<char>( ci->nameOff ), ci->nameLen ) ;
								nl += 1 + ci->nameLen ;
							}
						}
					}
					nameBuffer[nl] = '\0' ;
					int minLeft = t4_seq( cx, extendedOverlaps[0].seqIdx )->minLeftExtAnchor ;
					int minRight = t4_seq( cx, extendedOverlaps[lastEndExtendedOverlapIdx].seqIdx )->minRightExtAnchor ;
					// release the merged-away contigs (SeqSet::ReleaseSeq: the slot stays, NULL consensus)
					for ( i = 0 ; i < eOverlapCnt ; ++i )
					{
						int sIdx = extendedOverlaps[i].seqIdx ;
						if ( sIdx == newSeqIdx )
							continue ;
						T4Contig *c = t4_seq( cx, sIdx ) ;
						c->consOff = 0 ;
						c->pwOff = 0 ;
						c->nameOff = 0 ;
						c->len = 0 ;
					}
					ns->nameOff = nbOff ;
					ns->nameLen = nl ;
					ns->consOff = co ;
					ns->pwOff = po ;
					ns->cap = cap ;
					ns->lead = lead ;
					ns->len = newConsensusLen ;
					memcpy( t4_cons( cx, ns ), newConsensus, newConsensusLen ) ;
					s_update_consensus( cx, newSeqIdx, false ) ;
					s_build_index( cx, t4_cons( cx, ns ), newConsensusLen, newSeqIdx, barcode, 0 ) ;
					ns->minLeftExtAnchor = minLeft ;
					ns->minRightExtAnchor = minRight ;
					plan.readInConsensusOffset = 0 ;
					if ( extendedOverlaps[0].seqStart > 0 )
						plan.readInConsensusOffset = extendedOverlaps[0].seqStart ;
					plan.seqIdx = newSeqIdx ;
				}
			}
		}
	}
}

// The extend / inside commit (SeqSet.hpp:4131-4316) of the one extended overlap p.e0: grows its contig by the read's
// overhangs (index first, in the reference's order), decays the end weights and applies the scheduled consensus
// substitutions.  Collective.  Sets p.seqIdx and p.readInConsensusOffset, or p.ret and p.bail when the contig cannot
// grow.  Borrows tmpc (st->extOff, whose pre[] is dead after the decision) for the new left k-mers, and sm->bi[0 .. 9]
// for broadcasts within the phase.
T4_D inline void c_extend_commit( T4Ctx &cx, T4AddPlan &p, const char *r, int len, int barcode, int minKmerCount, char *tmpc )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	const T4Ovl &e0 = p.e0 ;
	const int seqIdx = e0.seqIdx ;
	p.seqIdx = seqIdx ;
	T4Contig *seq = t4_seq( cx, seqIdx ) ;
	if ( cx.tid == 0 )
		++seq->numRead ;
	if ( e0.readStart > 0 || e0.readEnd < len - 1 )
	{
		const int shift = e0.readStart ;
		const int rightAdd = ( e0.readEnd < len - 1 ) ? ( len - 1 - e0.readEnd ) : 0 ;
		const int oldLen = seq->len ;
		const int kl = st->kmerLength ;
		// index first, in the reference's order: new left k-mers, shift the old postings, (later) new right k-mers
		if ( shift > 0 )
		{
			char *oldCons = t4_cons( cx, seq ) ;
			// tmpc: newConsensus[0 .. shift + kl - 1): read prefix + the first kl-1 old bases
			int n = shift + kl - 1 ;
			T4_PAR_FOR( i, n )
			{
				char c ;
				if ( i < shift )
					c = r[i] ;
				else if ( i - shift < oldLen )
					c = oldCons[i - shift] ;
				else
				{
					int ri = e0.readEnd + 1 + ( i - shift - oldLen ) ;
					c = ( ri < len ) ? r[ri] : '\0' ;
				}
				tmpc[i] = c ;
			}
			T4_SYNC() ;
			c_index_op( cx, tmpc, n, T4_IDX_BUILD, seqIdx, barcode, 0, 0 ) ;
			c_index_op( cx, oldCons, oldLen, T4_IDX_UPDATE, seqIdx, barcode, shift, seqIdx ) ;
		}
		T4_SYNC() ; // every thread has read the old length / pointers
		if ( cx.tid == 0 )
			sm->bi[0] = s_contig_grow( cx, seq, shift, rightAdd ) ? 1 : 0 ;
		T4_SYNC() ;
		bool grown = sm->bi[0] != 0 ;
		T4_SYNC() ;
		if ( !grown )
		{
			p.ret = T4_E_NOMEM ;
			p.bail = true ;
		}
		else
		{
			char *newConsensus = t4_cons( cx, seq ) ;
			int *pw = t4_pw( cx, seq ) ;
			unsigned char *eq = t4_eq( cx, seq ) ;
			const int newConsensusLen = seq->len ;
			T4_PAR_FOR( i, shift )
				newConsensus[i] = r[i] ;
			T4_PAR_FOR( x, rightAdd )
				newConsensus[shift + oldLen + x] = r[e0.readEnd + 1 + x] ;
			T4_PAR_FOR( i, shift )
				t4_col_put( pw, eq, i, 0, 0, 0, 0 ) ;
			T4_PAR_FOR( i, rightAdd )
				t4_col_put( pw, eq, shift + oldLen + i, 0, 0, 0, 0 ) ;
			T4_SYNC() ;
			if ( e0.readEnd < len - 1 )
			{
				int start = e0.readStart + e0.seqEnd - kl + 2 ;
				if ( start < 0 )
				{
					if ( cx.tid == 0 )
						t4_raise( cx, T4_E_INTERNAL, 11 ) ;
					start = 0 ;
				}
				c_index_op( cx, newConsensus + start, newConsensusLen - start, T4_IDX_BUILD, seqIdx, barcode, start, 0 ) ;
			}
			// end-weight decay and scheduled consensus substitutions (SeqSet.hpp:4192-4247): four columns, serial
			if ( cx.tid == 0 )
			{
				int nrep = 0 ;
				if ( shift > 0 && ( barcode == -1 || minKmerCount > 1 ) )
				{
					for ( int i = 0 ; i < 2 ; ++i )
					{
						if ( i + shift >= len || r[i + shift] == 'N' )
							continue ;
						char nc = newConsensus[i + shift] ;
						if ( r[i + shift] != nc && nc != 'N' && pw[4 * ( i + shift ) + t4_nuc( nc )] == 1 )
						{
							sm->bi[2 + nrep] = i + shift ;
							sm->bi[6 + nrep] = r[i + shift] ;
							++nrep ;
						}
						for ( int j = 0 ; j < 4 ; ++j )
							if ( r[i + shift] != t4_numToNuc( j ) && pw[4 * ( i + shift ) + j] > 1 )
								t4_col_add( pw, eq, i + shift, j, -1 ) ;
					}
				}
				if ( e0.readEnd < len - 1 && ( barcode == -1 || minKmerCount > 1 ) )
				{
					for ( int i = oldLen - 2 ; i < oldLen ; ++i )
					{
						int pos = i - e0.seqStart ;
						int seqPos = i + shift ;
						if ( pos < 0 || r[pos] == 'N' )
							continue ;
						if ( i < 0 )
						{
							t4_raise( cx, T4_E_INTERNAL, 12 ) ;
							continue ;
						}
						char nc = newConsensus[seqPos] ;
						if ( r[pos] != nc && nc != 'N' && pw[4 * seqPos + t4_nuc( nc )] == 1 )
						{
							sm->bi[2 + nrep] = seqPos ;
							sm->bi[6 + nrep] = r[pos] ;
							++nrep ;
						}
						for ( int j = 0 ; j < 4 ; ++j )
							if ( r[pos] != t4_numToNuc( j ) && pw[4 * seqPos + j] > 1 )
								t4_col_add( pw, eq, seqPos, j, -1 ) ;
					}
				}
				if ( shift > 0 )
					seq->minLeftExtAnchor = 0 ;
				if ( e0.readEnd < len - 1 )
					seq->minRightExtAnchor = 0 ;
				sm->bi[1] = nrep ;
			}
			T4_SYNC() ;
			// (the +GENE name adjustment needs isRef overlaps: never in the stage-1 novel set, SeqSet.hpp:4258-4296)
			p.readInConsensusOffset = 0 ;
			if ( e0.seqStart > 0 )
				p.readInConsensusOffset = e0.seqStart ;
			int nrep = sm->bi[1] ;
			int repPos[4], repChar[4] ;
			for ( int i = 0 ; i < nrep ; ++i )
			{
				repPos[i] = sm->bi[2 + i] ;
				repChar[i] = sm->bi[6 + i] ;
			}
			T4_SYNC() ;
			for ( int i = 0 ; i < nrep ; ++i )
				c_substitute_consensus_pos( cx, seqIdx, repPos[i], (char)repChar[i] ) ;
		}
	}
	else
		p.readInConsensusOffset = e0.seqStart ;
}

// The posWeight update (SeqSet.hpp:4318-4363): adds the read to the columns of contig seqIdx from
// readInConsensusOffset on, then fills the consensus N's under the read and indexes their k-mers (thread 0; rare).
// Collective.  strand: the overlaps' strand.  Borrows nPos (st->extOff, whose pre[] is dead after the decision) for
// the read positions of those N's, and sm->bi[0] within the phase.
T4_D inline void c_posweight_update( T4Ctx &cx, int seqIdx, int readInConsensusOffset, const char *r, int len, int barcode, int strand,
	int *nPos )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	T4Contig *seq = t4_seq( cx, seqIdx ) ;
	char *cons = t4_cons( cx, seq ) ;
	int *pw = t4_pw( cx, seq ) ;
	unsigned char *eq = t4_eq( cx, seq ) ;
	if ( cx.tid == 0 )
		sm->bi[0] = 0 ;
	T4_SYNC() ;
	T4_PAR_FOR( i, len )
	{
		if ( r[i] == 'N' )
			continue ;
		t4_col_add( pw, eq, i + readInConsensusOffset, t4_nuc( r[i] ), 1 ) ;
		if ( cons[i + readInConsensusOffset] == 'N' )
			sm->bi[0] = 1 ;
	}
	T4_SYNC() ;
	if ( cx.tid == 0 )
	{
		t4_set_prev( st, seqIdx, 0, len - 1, readInConsensusOffset, strand ) ;
		if ( sm->bi[0] )
		{
			// consensus N's under the read are filled and their k-mers indexed (SeqSet.hpp:4338-4360); rare
			int kl = st->kmerLength ;
			int size = 0 ;
			for ( int i = 0 ; i < len ; ++i )
				if ( r[i] != 'N' && cons[i + readInConsensusOffset] == 'N' )
					nPos[size++] = i ;
			for ( int i = 0 ; i < size ; )
			{
				int j ;
				for ( j = i + 1 ; j < size ; ++j )
					if ( nPos[j] > nPos[j - 1] + kl - 1 )
						break ;
				for ( int l = i ; l < j ; ++l )
					cons[nPos[l] + readInConsensusOffset] = r[nPos[l]] ;
				int start = nPos[i] - kl + 1 + readInConsensusOffset ;
				if ( start < 0 )
					start = 0 ;
				int end = nPos[j - 1] + kl - 1 + readInConsensusOffset ;
				if ( end >= seq->len )
					end = seq->len - 1 ;
				s_build_index( cx, cons + start, end - start + 1, seqIdx, barcode, start ) ;
				i = j ;
			}
		}
	}
}

// SeqSet::AddRead (SeqSet.hpp:3426-4473), novel-contig set.  Collective; reads cx.sm->read / rc.
T4_D T4_BIG int c_add_read( T4Ctx &cx, int len, const char *geneName, int &strand, int barcode, int minKmerCount,
	bool repetitiveData, double similarityThreshold )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	if ( cx.tid == 0 )
		t4_set_prev( st, -1, -1, -1, -1, 0 ) ;
	int overlapCnt = c_get_overlaps( cx, len, strand, barcode, repetitiveData ) ;
	T4_PHASE( cx, 0 ) ;
	if ( st->error )
		return st->error ;
	if ( overlapCnt <= 0 )
		return -1 ;
	T4Ovl *overlaps = cx.P<T4Ovl>( st->ovlOff ) ;
	if ( geneName[0] != '\0' )
	{
		overlapCnt = c_gene_filter( cx, overlaps, overlapCnt, geneName ) ;
		if ( overlapCnt <= 0 )
			return -1 ;
	}
	c_sort_overlaps( cx, overlapCnt ) ;

	const char *r = ( overlaps[0].strand == 1 ) ? sm->read : sm->rc ;
	const double factor = ( barcode == -1 && !repetitiveData ) ? 1.0 : 2.0 ;
	T4Ovl *pre = cx.P<T4Ovl>( st->extOff ) ; // ExtendOverlap of every overlap; scratch of the commits after the decision
	T4_PHASE( cx, 5 ) ;
	long long xt[4] = { 0, 0, 0, 0 } ; // thread 0's clock64() around and inside the pass: counters 17-19
#if T4_CUDA
	xt[0] = clock64() ;
#endif
	const bool easy = c_extend_overlaps( cx, overlaps, overlapCnt, r, len, factor, similarityThreshold, pre, xt + 1 ) ;
#if T4_CUDA
	if ( cx.tid == 0 )
	{
		xt[3] = clock64() ;
		t4_count( cx, 17, (u64)( xt[1] - xt[0] ) ) ;
		t4_count( cx, 18, (u64)( xt[2] - xt[1] ) ) ;
		t4_count( cx, 19, (u64)( xt[3] - xt[2] ) ) ;
		t4_count( cx, 20, easy ? 1 : 0 ) ;
	}
#else
	(void)easy ;
#endif
	T4_PHASE( cx, 6 ) ;
	if ( cx.tid == 0 )
	{
		T4AddPlan &plan = sm->plan ;
		plan.kind = 0 ;
		plan.seqIdx = -1 ;
		plan.readInConsensusOffset = 0 ;
		plan.ret = -1 ;
		plan.bail = false ;
		plan.added = false ;
		T4Ovl *extendedOverlaps = cx.P<T4Ovl>( st->ovlTmpOff ) ;
		bool sortExtendedOverlaps ;
		const int k = s_decide_overlaps( cx, overlaps, overlapCnt, r, len, factor, pre, minKmerCount, similarityThreshold,
			extendedOverlaps, sortExtendedOverlaps ) ;
		if ( k > 1 )
			s_merge_commit( cx, extendedOverlaps, k, sortExtendedOverlaps, r, len, barcode, (int *)pre, plan ) ;
		else if ( k == 1 )
		{
			plan.added = true ;
			plan.kind = 1 ;
			plan.e0 = extendedOverlaps[0] ;
		}
	}
	T4_SYNC() ;
	T4AddPlan p = sm->plan ;
	if ( p.kind == 1 )
		c_extend_commit( cx, p, r, len, barcode, minKmerCount, (char *)pre ) ;
	if ( p.added && !p.bail && p.seqIdx >= 0 && !st->error )
	{
		c_posweight_update( cx, p.seqIdx, p.readInConsensusOffset, r, len, barcode, overlaps[0].strand, (int *)pre ) ;
		p.ret = p.seqIdx ;
	}
	// addNew is only kept for isRef overlaps (SeqSet.hpp:4377-4391): never in the novel set
	if ( p.ret == -1 && !p.bail )
	{
		if ( cx.tid == 0 )
			t4_set_prev( st, -2, -1, -1, -1, 0 ) ;
		p.ret = -2 ;
	}
	if ( p.ret >= 0 && strand == 0 )
		strand = overlaps[0].strand ;
	T4_SYNC() ;
	T4_PHASE( cx, 0 ) ;
	if ( st->error )
		return st->error ;
	return p.ret ;
}


// ---------------------------------------------------------------------------
// loading a read into shared memory
// ---------------------------------------------------------------------------
T4_D inline void c_load_read( T4Ctx &cx, const char *src, int len )
{
	T4Smem *sm = cx.sm ;
	T4_SYNC() ;
	T4_PAR_FOR( i, len )
	{
		char c = src[i] ;
		sm->read[i] = c ;
		sm->rc[len - 1 - i] = ( c != 'N' ) ? t4_numToNuc( 3 - t4_nuc( c ) ) : 'N' ;
	}
	if ( cx.tid == 0 )
	{
		sm->read[len] = '\0' ;
		sm->rc[len] = '\0' ;
		s_refill_slab( cx ) ;
	}
	T4_SYNC() ;
}

// The same from the 2-bit packed pool (t4_common.h): 2.7x fewer HBM bytes per read than ASCII and no revcomp pass.
T4_D inline void c_load_read_packed( T4Ctx &cx, const u64 *pk, int len )
{
	T4Smem *sm = cx.sm ;
	const int W = (int)t4_pack_w( len ) ;
	const u64 *fw = pk, *rc = pk + W ;
	const u32 *nm = (const u32 *)( pk + 2 * W ) ;
	T4_SYNC() ;
	T4_PAR_FOR( i, len )
	{
		const int sh = 62 - 2 * ( i & 31 ) ;
		const bool n = ( nm[i >> 5] >> ( i & 31 ) ) & 1u ;
		const int j = len - 1 - i ; // forward position of reverse-complement base i
		const bool nr = ( nm[j >> 5] >> ( j & 31 ) ) & 1u ;
		sm->read[i] = n ? 'N' : t4_numToNuc( (int)( ( fw[i >> 5] >> sh ) & 3 ) ) ;
		sm->rc[i] = nr ? 'N' : t4_numToNuc( (int)( ( rc[i >> 5] >> sh ) & 3 ) ) ;
	}
	if ( cx.tid == 0 )
	{
		sm->read[len] = '\0' ;
		sm->rc[len] = '\0' ;
		s_refill_slab( cx ) ;
	}
	T4_SYNC() ;
}

// ---------------------------------------------------------------------------
// the stage-1 driver loop (main.cpp:1583-1881) and rescue pass (main.cpp:1897-1940) over read descriptors
// ---------------------------------------------------------------------------
T4_D inline double t4_rescue_threshold( int minCnt )
{
	double t = 0.9 ;
	if ( minCnt >= 20 )
		t = 0.97 ;
	else if ( minCnt >= 2 )
		t = 0.95 ;
	return t ;
}

// main.cpp:1782-1843: a read that was added and annotates well marks its mate (and the mate's identical copies) as a
// good candidate for a motif-anchored new contig.  Thread 0.
T4_D inline void s_mate_hint( const t4_read_desc *descs, int n, int i, int mateIdx, u32 flags, int finalStrand, int8_t *goodCandidate,
	int32_t *info )
{
	bool good = false ;
	if ( finalStrand == 1 && ( flags & T4_RD_GOOD_PLUS ) )
		good = true ;
	if ( finalStrand == -1 && ( flags & T4_RD_GOOD_MINUS ) )
		good = true ;
	if ( good && !goodCandidate[mateIdx] )
	{
		int tagm = mateIdx ;
		const t4_read_desc &md = descs[tagm] ;
		for ( int j = tagm - 1 ; j > 0 && j >= md.eq_lo ; --j )
		{
			goodCandidate[j] = 1 ;
			info[j] = i ;
		}
		for ( int j = tagm + 1 ; j < n && j < md.eq_hi ; ++j )
		{
			goodCandidate[j] = 1 ;
			info[j] = i ;
		}
	}
	if ( good )
	{
		goodCandidate[mateIdx] = 1 ;
		info[mateIdx] = i ;
	}
}

T4_D inline void c_run_loop( T4Ctx &cx, T4Op *op, const int *gapLimitTable )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	const t4_read_desc *descs = t4_x<t4_read_desc>( op->desc ) ;
	const char *pool = t4_x<char>( op->pool ) ;
	T4Names *names = t4_x<T4Names>( op->names ) ;
	const char *namePool = t4_x<char>( names->pool ) ;
	const u32 *nameOff = t4_x<u32>( names->off ) ;
	int32_t *retCodes = t4_x<int32_t>( op->retCodes ) ;
	int8_t *strands = t4_x<int8_t>( op->strands ) ;
	int32_t *rescueRet = t4_x<int32_t>( op->rescueRet ) ;
	int32_t *rescueList = t4_x<int32_t>( op->rescueList ) ;
	int8_t *goodCandidate = t4_x<int8_t>( op->good ) ;
	int32_t *info = t4_x<int32_t>( op->info ) ;
	const t4_run_cfg cfg = op->cfg ;
	const int n = op->n ;
	const u64 *packed = t4_x<u64>( op->packed ) ;
	const u64 packStride = op->packStride ;
	uint8_t *events = t4_x<uint8_t>( op->events ) ;
	T4_PAR_FOR( i, n )
	{
		goodCandidate[i] = 0 ;
		info[i] = -1 ;
		rescueRet[i] = INT32_MIN ;
	}
	T4_SYNC() ;
	// barcodeTotalReadCount (main.cpp:1572-1581), only when finished barcodes are purged
	T4BcTable bc ;
	bc.cap = 0 ;
	const bool releaseBarcodes = cfg.has_barcode && cfg.release_barcodes && n > 0 ;
	if ( releaseBarcodes )
	{
		u32 cap = 16 ;
		while ( cap < 2u * (u32)n )
			cap *= 2 ;
		if ( cx.tid == 0 )
			sm->bu[0] = s_alloc( cx, (u64)cap * 16 ) ;
		T4_SYNC() ;
		u64 off = sm->bu[0] ;
		T4_SYNC() ;
		if ( !off )
			return ;
		bc.cap = cap ;
		bc.key = cx.P<u64>( off ) ;
		bc.total = (u32 *)( bc.key + cap ) ;
		bc.done = bc.total + cap ;
		T4_PAR_FOR( i, cap )
		{
			bc.key[i] = 0 ;
			bc.total[i] = 0 ;
			bc.done[i] = 0 ;
		}
		T4_SYNC() ;
		T4_PAR_FOR( i, n )
			if ( descs[i].barcode != -1 )
				t4_atomic_add32( &bc.total[t4_bc_slot( bc, descs[i].barcode, true )], 1 ) ;
		T4_SYNC() ;
	}
	int assembledReadCnt = 0 ;
	int prevAddRet = -1 ;
	int indexKmerLength = st->kmerLength ;
	int changeKmerLengthThreshold = cfg.change_k_threshold ;
	int rescueCnt = 0 ;
	int dupCredit = 0 ; // upcoming duplicate records whose RepeatAddRead increments are already applied
	for ( int i = 0 ; i < n && !st->error ; ++i )
	{
		const t4_read_desc d = descs[i] ;
		int addRet = -1 ;
		const bool credited = ( d.flags & T4_RD_DUP ) && dupCredit > 0 ;
		int batchExtra = 0 ;
		if ( d.len > T4_DEV_MAX_READ || d.len < 0 )
		{
			if ( cx.tid == 0 )
				t4_raise( cx, T4_E_UNSUPPORTED, 4 ) ;
			T4_SYNC() ;
			break ;
		}
		if ( credited )
			; // same read string as the record before: nothing to load, nothing to add
		else if ( packed )
			c_load_read_packed( cx, packed + (u64)i * packStride, d.len ) ;
		else
			c_load_read( cx, pool + d.seq_off, d.len ) ;
		int finalStrand = 0 ;
		u32 ev = 0 ;
		if ( !( d.flags & T4_RD_DUP ) )
		{
			int strand = 0 ;
			if ( !( d.flags & T4_RD_FILTERED ) )
			{
				ev |= T4_EV_ADD_READ ;
				char name[5] ;
				name[0] = d.gene4[0] ; name[1] = d.gene4[1] ; name[2] = d.gene4[2] ; name[3] = d.gene4[3] ; name[4] = '\0' ;
				strand = d.strand_in ;
				addRet = c_add_read( cx, d.len, name, strand, d.barcode, d.min_kmer_count, cfg.repetitive != 0, d.sim_threshold ) ;
				if ( st->error )
					break ;
				if ( addRet < 0 )
				{
					int novelStrand = 0 ;
					const char *nm = 0 ;
					int nmLen = 0 ;
					if ( d.flags & T4_RD_NOVEL_ON_FAIL )
					{
						ev |= T4_EV_NOVEL_ANCHORED ;
						novelStrand = d.novel_strand ;
						nm = namePool + nameOff[d.name_id] ;
						nmLen = (int)( nameOff[d.name_id + 1] - nameOff[d.name_id] ) ;
					}
					else if ( d.flags & T4_RD_MOTIF_FORCED )
					{
						if ( d.novel_strand != 0 && ( d.flags & T4_RD_MOTIF ) )
						{
							ev |= T4_EV_NOVEL_MOTIF ;
							novelStrand = d.novel_strand ;
							nm = "Novel" ;
							nmLen = 5 ;
						}
					}
					else if ( goodCandidate[i] )
					{
						int ms = -strands[info[i]] ;
						if ( ms != 0 && ( d.flags & T4_RD_MOTIF ) )
						{
							ev |= T4_EV_NOVEL_MOTIF ;
							novelStrand = ms ;
							nm = "Novel" ;
							nmLen = 5 ;
						}
					}
					if ( nm != 0 )
					{
						T4_PHASE( cx, 7 ) ;
						addRet = c_input_novel_read( cx, nm, nmLen, d.len, novelStrand, d.barcode ) ;
						T4_PHASE( cx, 0 ) ;
					}
				}
			}
			finalStrand = ( d.flags & T4_RD_FILTERED ) ? 0 : strand ;
		}
		else
		{
			T4_PHASE( cx, 7 ) ;
			if ( prevAddRet != -1 && prevAddRet != -3 )
			{
				ev |= T4_EV_REPEAT ;
				if ( credited )
				{
					addRet = st->prevSeqIdx ;
					--dupCredit ;
				}
				else
				{
					// A run of L duplicate records is L RepeatAddRead calls on unchanged prevAddInfo: apply them in one pass.
					// L stops where the loop could act between two of them: at the record that makes assembledReadCnt a
					// multiple of update_consensus_every (UpdateAllConsensus must see exactly the counts of the records so
					// far, main.cpp:1862), and it is 1 when a k change is pending (ChangeKmerLength resets prevAddInfo).
					int L = 1 ;
					const bool kPending = changeKmerLengthThreshold > 0 && st->nSeqs > changeKmerLengthThreshold && indexKmerLength < 16
						&& !cfg.has_barcode ;
					if ( st->prevSeqIdx >= 0 && !kPending )
					{
						L = c_dup_run_len( cx, descs, i, n, 4096 ) ;
						if ( cfg.update_consensus_every > 0 && !cfg.has_barcode )
						{
							const int room = cfg.update_consensus_every - ( assembledReadCnt % cfg.update_consensus_every ) ;
							if ( L > room )
								L = room ;
						}
						if ( L < 1 )
							L = 1 ;
					}
					addRet = c_repeat_add_read_n( cx, d.len, L ) ;
					if ( releaseBarcodes )
						dupCredit = L - 1 ; // the purge bookkeeping stays per record
					else
						batchExtra = L - 1 ; // the other L - 1 records are closed right below, without a loop iteration each
				}
			}
			else if ( prevAddRet == -3 )
				addRet = -3 ;
			T4_PHASE( cx, 0 ) ;
			finalStrand = i > 0 ? strands[i - 1] : 0 ;
		}
		if ( cx.tid == 0 )
		{
			strands[i] = (int8_t)finalStrand ;
			retCodes[i] = addRet ;
			if ( addRet == -2 )
				rescueList[rescueCnt] = i ;
			else if ( addRet >= 0 && d.mate_idx > i )
				s_mate_hint( descs, n, i, d.mate_idx, d.flags, finalStrand, goodCandidate, info ) ;
		}
		if ( addRet == -2 )
			++rescueCnt ;
		else if ( addRet >= 0 )
			++assembledReadCnt ;
		T4_SYNC() ;
		if ( batchExtra > 0 )
		{
			// records i + 1 .. i + batchExtra: duplicates whose RepeatAddRead is already applied (addRet >= 0, same strand)
			for ( int t = cx.tid ; t < batchExtra ; t += cx.nt )
			{
				retCodes[i + 1 + t] = addRet ;
				strands[i + 1 + t] = (int8_t)finalStrand ;
				if ( events )
					events[i + 1 + t] = (uint8_t)T4_EV_REPEAT ;
			}
			if ( cx.tid == 0 )
				for ( int t = 0 ; t < batchExtra ; ++t )
				{
					const int idx = i + 1 + t ;
					const int mi = descs[idx].mate_idx ;
					if ( mi > idx )
						s_mate_hint( descs, n, idx, mi, descs[idx].flags, finalStrand, goodCandidate, info ) ;
				}
			assembledReadCnt += batchExtra ;
			if ( events && cx.tid == 0 )
				events[i] = (uint8_t)ev ; // the head record's own byte (the loop end writes index i + batchExtra)
			i += batchExtra ;
			ev = T4_EV_REPEAT ;
			T4_SYNC() ;
		}
		// main.cpp:1846-1859 (inside `else if ( addRet >= 0 )`): a barcode is finished when as many of its reads were
		// assembled as it has reads
		if ( releaseBarcodes && addRet >= 0 && d.barcode != -1 )
		{
			if ( cx.tid == 0 )
			{
				u32 sl = t4_bc_slot( bc, d.barcode, false ) ;
				sm->bi[0] = ( sl != 0xffffffffu && ++bc.done[sl] >= bc.total[sl] ) ? 1 : 0 ;
			}
			T4_SYNC() ;
			const bool fin = sm->bi[0] != 0 ;
			T4_SYNC() ;
			if ( fin )
			{
				ev |= T4_EV_PURGED ;
				T4_PHASE( cx, 7 ) ;
				c_release_barcode( cx, d.barcode, cfg.contig_min_cov ) ;
				T4_PHASE( cx, 0 ) ;
			}
		}
		if ( assembledReadCnt > 0 && cfg.update_consensus_every > 0 && assembledReadCnt % cfg.update_consensus_every == 0
			&& !cfg.has_barcode )
		{
			T4_PHASE( cx, 7 ) ;
			c_update_all_consensus( cx ) ;
			T4_PHASE( cx, 0 ) ;
		}
		prevAddRet = addRet ;
		if ( changeKmerLengthThreshold > 0 && st->nSeqs > changeKmerLengthThreshold && indexKmerLength < 16 && !cfg.has_barcode )
		{
			changeKmerLengthThreshold *= 4 ;
			indexKmerLength += 2 ;
			ev |= T4_EV_CHANGE_K ;
			c_change_kmer_length( cx, indexKmerLength, gapLimitTable[indexKmerLength] ) ;
		}
		if ( events && cx.tid == 0 )
			events[i] = (uint8_t)ev ;
	}
	T4_PHASE( cx, 7 ) ;
	if ( cfg.final_update && !st->error )
		c_update_all_consensus( cx ) ;
	T4_PHASE( cx, 0 ) ;
	if ( cfg.do_rescue && cfg.first_read_len <= 200 && !st->error )
	{
		for ( int x = 0 ; x < rescueCnt && !st->error ; ++x )
		{
			int i = rescueList[x] ;
			const t4_read_desc d = descs[i] ;
			if ( packed )
				c_load_read_packed( cx, packed + (u64)i * packStride, d.len ) ;
			else
				c_load_read( cx, pool + d.seq_off, d.len ) ;
			char name[2] = "" ;
			int strand = 0 ;
			int addRet = c_add_read( cx, d.len, name, strand, d.barcode, 1, cfg.repetitive != 0, t4_rescue_threshold( d.min_cnt ) ) ;
			if ( cx.tid == 0 )
			{
				strands[i] = (int8_t)strand ;
				rescueRet[i] = addRet ;
				if ( events )
					events[i] |= T4_EV_RESCUED ;
			}
			T4_SYNC() ;
		}
		if ( cfg.final_update && !st->error )
			c_update_all_consensus( cx ) ;
	}
	if ( cx.tid == 0 )
	{
		st->assembledReadCnt = assembledReadCnt ;
		st->prevAddRet = prevAddRet ;
		t4_count( cx, 0, (u64)n ) ;
	}
	T4_SYNC() ;
}

// ---------------------------------------------------------------------------
// stream construction: SeqSet::SeqSet(int kl) (SeqSet.hpp:2558-2576)
// ---------------------------------------------------------------------------
T4_HD inline u64 t4_al( u64 x ) { return ( x + 63 ) & ~63ull ; }

T4_HD inline u64 t4_stream_footprint( const T4InitParams &ip )
{
	u64 o = t4_al( sizeof( T4Stream ) ) ;
	o += t4_al( (u64)ip.seqCap * sizeof( T4Contig ) ) ;
	o += t4_al( (u64)ip.dirCap * sizeof( T4Dir ) ) ;
	o += 2 * t4_al( (u64)ip.hitCap * 8 ) ;
	o += 2 * t4_al( (u64)( ip.hitCap + 1 ) * 4 ) ;
	o += t4_al( 2ull * T4_DEV_MAX_READ * sizeof( T4Pos ) ) ;
	o += 4 * t4_al( (u64)ip.ovlCap * sizeof( T4Ovl ) ) ;
	o += t4_al( (u64)ip.ovlCap * 8 ) ;
	o += t4_al( (u64)ip.ovlCap * 32 * 4 ) ;
	o += t4_al( (u64)ip.nThreads * T4_DP_STRIDE ) ;
	return o ;
}

T4_D inline void c_init_stream( T4Ctx &cx, u64 base, const T4InitParams &ip )
{
	T4Stream *st = cx.P<T4Stream>( base ) ;
	if ( cx.tid == 0 )
	{
		u64 o = base + t4_al( sizeof( T4Stream ) ) ;
		memset( st, 0, sizeof( T4Stream ) ) ;
		st->kmerLength = ip.kmerLength ;
		st->radius = 10 ;
		st->hitLenRequired = ip.hitLenRequired ;
		st->nomatchGapLimit = ip.nomatchGapLimit ;
		st->isLongSeqSet = 0 ;
		st->considerBarcode = ip.considerBarcode ;
		st->novelSeqSimilarity = 0.9 ;
		st->repeatSimilarity = 0.95 ;
		st->nSeqs = 0 ;
		st->seqCap = (int)ip.seqCap ;
		st->seqsOff = o ; o += t4_al( (u64)ip.seqCap * sizeof( T4Contig ) ) ;
		st->dirOff = o ; o += t4_al( (u64)ip.dirCap * sizeof( T4Dir ) ) ;
		st->dirCap = ip.dirCap ;
		st->dirUsed = 0 ;
		st->prevSeqIdx = -1 ;
		st->prevReadStart = -1 ;
		st->prevReadEnd = st->prevSeqStart = -1 ;
		st->prevStrand = 0 ;
		st->keysAOff = o ; o += t4_al( (u64)ip.hitCap * 8 ) ;
		st->keysBOff = o ; o += t4_al( (u64)ip.hitCap * 8 ) ;
		st->grpOff = o ; o += t4_al( (u64)( ip.hitCap + 1 ) * 4 ) ;
		st->runOff = o ; o += t4_al( (u64)( ip.hitCap + 1 ) * 4 ) ;
		st->hitCap = ip.hitCap ;
		st->posOff = o ; o += t4_al( 2ull * T4_DEV_MAX_READ * sizeof( T4Pos ) ) ;
		st->ovlOff = o ; o += t4_al( (u64)ip.ovlCap * sizeof( T4Ovl ) ) ;
		st->ovlTmpOff = o ; o += t4_al( (u64)ip.ovlCap * sizeof( T4Ovl ) ) ;
		st->extOff = o ; o += t4_al( (u64)ip.ovlCap * sizeof( T4Ovl ) ) ;
		st->failOff = o ; o += t4_al( (u64)ip.ovlCap * sizeof( T4Ovl ) ) ;
		st->anchorOff = o ; o += t4_al( (u64)ip.ovlCap * 8 ) ;
		st->bitsOff = o ; o += t4_al( (u64)ip.ovlCap * 32 * 4 ) ;
		st->ovlCap = ip.ovlCap ;
		st->dpOff = o ; o += t4_al( (u64)ip.nThreads * T4_DP_STRIDE ) ;
		st->dpStride = T4_DP_STRIDE ;
		st->nThreads = ip.nThreads ;
		st->prevAddRet = -1 ;
	}
	T4Dir *dir = cx.P<T4Dir>( base + t4_al( sizeof( T4Stream ) ) + t4_al( (u64)ip.seqCap * sizeof( T4Contig ) ) ) ;
	T4_PAR_FOR( i, ip.dirCap )
	{
		dir[i].key = 0 ;
		dir[i].listOff = 0 ;
		dir[i].cnt = dir[i].cap = dir[i].lock = dir[i].pad = 0 ;
	}
	T4_SYNC() ;
}

// t4_init_kernel: block b lays out the b-th stream from base on, ip.footprint bytes apart
T4_D inline void c_init_block( char *A, u64 base, const T4InitParams &ip, u32 b, int tid, int nt )
{
	T4Ctx cx = t4_ctx( A, 0, 0, tid, nt ) ;
	c_init_stream( cx, base + (u64)b * ip.footprint, ip ) ;
}

// ---------------------------------------------------------------------------
// op dispatch: body of the stream kernel (one CTA = one T4Op)
// ---------------------------------------------------------------------------
T4_D inline void c_run_op( T4Ctx &cx, T4Op *op, const int *gapLimitTable )
{
	T4Stream *st = cx.st ;
	T4Smem *sm = cx.sm ;
	if ( st->error )
	{
		if ( cx.tid == 0 )
			op->ret = st->error ;
		return ;
	}
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
	switch ( op->op )
	{
		case T4_OP_RUN_LOOP:
			c_run_loop( cx, op, gapLimitTable ) ;
			if ( cx.tid == 0 )
				op->ret = st->error ? st->error : st->assembledReadCnt ;
			break ;
		case T4_OP_ADD_READ:
		{
			c_load_read( cx, t4_x<char>( op->read ), op->len ) ;
			int strand = op->strand ;
			int ret = c_add_read( cx, op->len, op->gene, strand, op->barcode, op->minKmerCount, op->repetitive != 0, op->thr ) ;
			if ( cx.tid == 0 )
			{
				op->ret = ret ;
				op->strandOut = strand ;
			}
			break ;
		}
		case T4_OP_REPEAT:
		{
			c_load_read( cx, t4_x<char>( op->read ), op->len ) ;
			int ret = c_repeat_add_read( cx, op->len ) ;
			if ( cx.tid == 0 )
				op->ret = ret ;
			break ;
		}
		case T4_OP_INPUT_NOVEL:
		{
			c_load_read( cx, t4_x<char>( op->read ), op->len ) ;
			int r0 = c_input_novel_read( cx, t4_x<char>( op->name ), op->nameLen, op->len, op->strand, op->barcode ) ;
			if ( cx.tid == 0 )
				op->ret = r0 ;
			break ;
		}
		case T4_OP_UPDATE_ALL:
			c_update_all_consensus( cx ) ;
			if ( cx.tid == 0 )
				op->ret = 0 ;
			break ;
		case T4_OP_CHANGE_K:
			c_change_kmer_length( cx, op->kl, gapLimitTable[op->kl] ) ;
			if ( cx.tid == 0 )
				op->ret = 0 ;
			break ;
		case T4_OP_RELEASE_BARCODE:
			c_release_barcode( cx, op->barcode, op->minKmerCount ) ;
			if ( cx.tid == 0 )
				op->ret = 0 ;
			break ;
		case T4_OP_RELEASE_SHALLOW:
			c_release_shallow( cx, op->minKmerCount ) ;
			if ( cx.tid == 0 )
				op->ret = 0 ;
			break ;
		case T4_OP_GET_HITS:
		{
			// GetHitsFromRead + SortHits, reported in (strand, idx, a, b) order as int32[5]
			c_load_read( cx, t4_x<char>( op->read ), op->len ) ;
			int ret = 0 ;
			if ( op->len >= st->kmerLength )
			{
				int anyBig = 0 ;
				u32 H = c_get_hits( cx, op->len, op->strand, op->barcode, op->repetitive != 0, &anyBig ) ;
				u64 *a = cx.P<u64>( st->keysAOff ) ;
				u64 *b = cx.P<u64>( st->keysBOff ) ;
				// re-key to SortHits order: (strand, idx, a, b)
				const T4Pos *pos = cx.P<T4Pos>( st->posOff ) ;
				const int m = op->len - st->kmerLength + 1 ;
				T4_PAR_FOR( i, H )
				{
					u64 kx = a[i] ;
					if ( kx == T4_KEY_INVALID )
						continue ;
					u64 aa = (u64)t4_key_a( kx ) ;
					a[i] = ( kx & ( ~0ull << T4_KEY_IDX_SHIFT ) ) | ( aa << 30 ) | ( (u64)t4_key_b( kx ) << 1 ) | ( kx & 1 ) ;
				}
				T4_SYNC() ;
				u64 *sorted = c_sort_keys( cx, a, b, H ) ;
				int32_t *out = t4_x<int32_t>( op->out ) ;
				T4_PAR_FOR( i, H )
				{
					u64 kx = sorted[i] ;
					if ( kx == T4_KEY_INVALID || i >= op->outCap )
						continue ;
					int strand = t4_key_strand( kx ) ;
					int aa = (int)( ( kx >> 30 ) & 0x7ff ) ;
					int bb = (int)( ( kx >> 1 ) & T4_KEY_B_MASK ) ;
					out[5 * i] = t4_key_idx( kx ) ;
					out[5 * i + 1] = bb ;
					out[5 * i + 2] = aa ;
					out[5 * i + 3] = strand ;
					int rep = (int)pos[( strand == 1 ? 0 : 1 ) * T4_DEV_MAX_READ + aa].cnt ;
					out[5 * i + 4] = ( op->barcode != -1 ) ? 1 : rep ;
				}
				T4_SYNC() ;
				u32 c = 0 ;
				for ( u32 i = cx.tid ; i < H ; i += cx.nt )
					if ( sorted[i] != T4_KEY_INVALID )
						++c ;
				u32 total ;
				c_scan_threads( cx, c, total ) ;
				ret = (int)total ;
				(void)m ;
			}
			if ( cx.tid == 0 )
				op->ret = ret ;
			break ;
		}
		case T4_OP_GET_OVERLAPS:
		{
			c_load_read( cx, t4_x<char>( op->read ), op->len ) ;
			int n = c_get_overlaps( cx, op->len, op->strand, op->barcode, op->repetitive != 0 ) ;
			if ( n > 0 )
			{
				T4Ovl *ovl = cx.P<T4Ovl>( st->ovlOff ) ;
				int32_t *out = t4_x<int32_t>( op->out ) ;
				double *sim = t4_x<double>( op->out2 ) ;
				T4_PAR_FOR( i, n )
				{
					if ( i >= op->outCap )
						continue ;
					out[8 * i] = ovl[i].seqIdx ;
					out[8 * i + 1] = ovl[i].readStart ;
					out[8 * i + 2] = ovl[i].readEnd ;
					out[8 * i + 3] = ovl[i].seqStart ;
					out[8 * i + 4] = ovl[i].seqEnd ;
					out[8 * i + 5] = ovl[i].strand ;
					out[8 * i + 6] = ovl[i].matchCnt ;
					out[8 * i + 7] = ovl[i].indelCnt ;
					sim[i] = ovl[i].similarity ;
				}
			}
			if ( cx.tid == 0 )
				op->ret = n ;
			break ;
		}
		default:
			break ;
	}
	T4_SYNC() ;
	if ( cx.tid == 0 && st->error && op->ret >= T4_E_BASE )
		op->ret = st->error ;
	T4_SYNC() ;
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
		{
			t4_atomic_add( &cx.g->counters[8 + i], (u64)sm->ph[i] ) ;
			tot += (u64)sm->ph[i] ;
		}
		st->nReads = tot ; // clock cycles this op took on this stream (diagnostics: t4_streams_cycles)
	}
#endif
	(void)sm ;
}

#endif
