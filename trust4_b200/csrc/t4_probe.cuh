// Grid-wide k-mer probe over FROZEN sets: SeqSet::GetHitsFromRead (SeqSet.hpp:1341-1501) + KmerIndex::Search
// (KmerIndex.hpp:104-116) for a whole batch of reads, one WARP per read, persistent CTAs.
//
// The stream kernel (t4_engine.h, one CTA per SeqSet) has to run its reads in order because AddRead mutates the set.
// A read-only pass has no such constraint: every read of the batch is independent, so the probe is laid out for
// memory-level parallelism instead of for serial latency --
//   * reads arrive 2-bit packed (t4_common.h) and are visited in (set, length-bucket) order (t4_bucket_kernel): the
//     warps of a CTA see equal work and consecutive warps hit the same directory, which keeps it in L2;
//   * a k-mer is one funnel shift of two packed words; each lane owns up to 9 positions of the read and issues
//     their directory probes back to back, one 32-byte T4Dir sector (two 128-bit loads) each;
//   * hit slots are a warp prefix sum over the postings counts; the >= 100-postings skip rule and the stale
//     prevKmerCode quirk (SeqSet.hpp:1376-1392) only exist when some list has >= 100 postings -- then the warp runs
//     the reference's state machine over shuffled (code, size) pairs instead;
//   * postings: lists of <= 4 entries are one sector (T4_ALIGN 32) and are fetched by their owner lane as one
//     sector; longer lists are pulled into shared memory by the TMA engine (cp.async.bulk + mbarrier, every
//     owner lane issues its own copies, all of a read's lists in flight at once) and converted to hit keys by the
//     whole warp with coalesced 8-byte stores; lists beyond the staging tile stream through 128-bit loads;
//   * the output range of a read is reserved with one atomicAdd, so hits of all reads form one dense key array.
// The keys are bit-identical to what c_get_hits() writes for the same read (same layout, same order).
#ifndef T4_PROBE_CUH
#define T4_PROBE_CUH

#if T4_CUDA

#define T4P_WARPS 1                 // warps per CTA: one, so that the warp's shared-memory tile sits at a constant address
                                    // (with 8 warps per CTA 18 % of all issued instructions recomputed `smem + warp * sizeof`)
#define T4P_PMAX 9                  // positions per lane and tile
#define T4P_TILE ( 32 * T4P_PMAX )  // positions (both strand passes) per tile: a 150 bp read at k = 9 has 284
#define T4P_STG 448                 // TMA staging tile per warp, postings (3.5 KB: 24 one-warp CTAs of 8.4 KB + 1 KB reserved fit an SM)
#define T4P_SHORT 4                 // a list of <= 4 postings is one 32-byte sector
#define T4P_TMA_MAX 256             // longer lists stream through 128-bit loads instead of the staging tile
#define T4P_NONE 0xffffffffu

struct T4ProbeParams
{
	char *A ;                  // arena
	const u64 *streamOff ;     // [nSets] arena offsets of the T4Stream records
	const t4_read_desc *descs ;
	const u64 *packed ;        // packed read pool: read i at packed + i * packStride
	u64 packStride ;
	const u64 *ord ;           // [nReads] read index | set index << 32, in (set, length bucket) order
	i64 nReads ;
	u64 *keys ;                // hit keys, dense
	u64 keyCap ;
	u64 *hitOff ;              // [nReads] first key of read i
	u32 *hitCnt ;              // [nReads] number of keys (invalid keys of the barcode filter included)
	u32 *hitFlags ;            // [nReads] bit 0: a k-mer has > 10000 postings (SeqSet.hpp:799), bit 1: serial rule path taken
	u64 *ctrl ;                // [0] read cursor [1] key cursor [2] overflow [3] lookups [4] postings [5] hits [6] packed read bytes [7] unsupported reads
	int allowTotalSkip ;
} ;

struct __align__( 16 ) T4ProbeWarp // sizeof is a multiple of 16: every warp's staging tile is a legal TMA destination
{
	u64 stg[T4P_STG] ;         // 16-byte aligned TMA destination
	u32 lo[T4P_TILE] ;         // per position of the tile: postings list offset >> 5 (lists are 32-byte aligned) ...
	u32 cnt[T4P_TILE] ;        // ... its length (0: k-mer with an N, pass not probed, code absent) ...
	u32 base[T4P_TILE] ;       // ... first hit slot of the read, T4P_NONE = lookup not taken
	u32 sb[T4P_TILE] ;         // table of the tile's TMA-staged lists: position index per entry, in position order
	u64 fw[18], rc[18] ;       // packed words (+ zero padding for the two-word funnel shift)
	u32 nm[20] ;
	u64 bar ;                  // mbarrier
} ;

__device__ __forceinline__ u64 t4p_extract( const u64 *W, int q, int k )
{
	const int w = q >> 5, s = ( q & 31 ) * 2 ;
	const u64 hi = W[w], lo = W[w + 1] ;
	const u64 v = s ? ( ( hi << s ) | ( lo >> ( 64 - s ) ) ) : hi ;
	return v >> ( 64 - 2 * k ) ;
}

__device__ __forceinline__ bool t4p_has_n( const u32 *M, int p, int k )
{
	const int w = p >> 5, s = p & 31 ;
	u32 v = M[w] >> s ;
	if ( s )
		v |= M[w + 1] << ( 32 - s ) ;
	return ( v & ( ( 1u << k ) - 1u ) ) != 0 ;
}

// One 32-byte sector.  sm_90 has no 256-bit load: two 128-bit loads of the same sector, issued back to back.
__device__ __forceinline__ void t4p_ld256( const void *p, u64 &a, u64 &b, u64 &c, u64 &d )
{
	asm volatile( "ld.global.nc.v2.u64 {%0,%1}, [%4];\n\t"
		      "ld.global.nc.v2.u64 {%2,%3}, [%4+16];"
		      : "=l"( a ), "=l"( b ), "=l"( c ), "=l"( d ) : "l"( p ) ) ;
}
__device__ __forceinline__ void t4p_ld128( const void *p, u64 &a, u64 &b )
{
	asm volatile( "ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"( a ), "=l"( b ) : "l"( p ) ) ;
}

__device__ __forceinline__ u32 t4p_smem( const void *p ) { return (u32)__cvta_generic_to_shared( p ) ; }

__device__ __forceinline__ void t4p_bar_init( u64 *bar )
{
	asm volatile( "mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"( t4p_smem( bar ) ) ) ;
	asm volatile( "fence.mbarrier_init.release.cluster;" ::: "memory" ) ;
}
__device__ __forceinline__ void t4p_bar_expect( u64 *bar, u32 bytes )
{
	asm volatile( "mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"( t4p_smem( bar ) ), "r"( bytes ) : "memory" ) ;
}
__device__ __forceinline__ void t4p_bar_wait( u64 *bar, u32 parity )
{
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"T4P_WAIT:\n"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
		"@p bra T4P_DONE;\n"
		"bra T4P_WAIT;\n"
		"T4P_DONE:\n"
		"}\n" ::"r"( t4p_smem( bar ) ),
		"r"( parity )
		: "memory" ) ;
}
// TMA bulk copy global -> shared (non-tensor form): 16-byte aligned source / destination, size a multiple of 16
__device__ __forceinline__ void t4p_bulk_g2s( void *dst, const void *src, u32 bytes, u64 *bar )
{
	asm volatile( "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"( t4p_smem( dst ) ),
		"l"( src ), "r"( bytes ), "r"( t4p_smem( bar ) )
		: "memory" ) ;
}

__device__ __forceinline__ u32 t4p_warp_excl_scan( u32 v, u32 &total, int lane )
{
	u32 inc = v ;
#pragma unroll
	for ( int d = 1 ; d < 32 ; d <<= 1 )
	{
		u32 t = __shfl_up_sync( 0xffffffffu, inc, d ) ;
		if ( lane >= d )
			inc += t ;
	}
	total = __shfl_sync( 0xffffffffu, inc, 31 ) ;
	return inc - v ;
}

// per-read constants
struct T4ProbeRead
{
	const T4Dir *dir ;
	u32 dirMask ;
	u64 salt ;                 // barcode salt of the directory key (t4_index_key)
	u64 mask ;                 // 2k low bits
	int k, len, m, strand, barcode, nPos ; // nPos = 2 m positions: forward pass [0, m), reverse-complement pass [m, 2 m)
	bool anyN ;                // the read holds an 'N' (otherwise every k-mer is valid and the mask test is skipped)
} ;

// Serial rule state (SeqSet.hpp:1376-1392, 1441-1455), carried across tiles and from the forward into the reverse pass.
struct T4ProbeScan
{
	u64 prev ;
	int skipCnt, curPass ;
	u32 total, lookups ;
	int big ;
} ;

__device__ __forceinline__ bool t4p_active( const T4ProbeRead &R, int x, int &pass, int &q )
{
	pass = x >= R.m ;
	q = pass ? x - R.m : x ;
	return x < R.nPos && !( ( pass == 0 && R.strand == -1 ) || ( pass == 1 && R.strand == 1 ) ) ;
}

__device__ __forceinline__ u64 t4p_base_at( const u64 *W, int p ) { return ( W[p >> 5] >> ( 62 - 2 * ( p & 31 ) ) ) & 3ull ; }

#define T4P_TAKEN 0x80000000u       // bit 31 of sw->cnt[i]: the position passes the plain "taken" predicate
#define T4P_CNT( v ) ( ( v ) & 0x7fffffffu )

// Directory probes of one tile.  Position i of the tile belongs to lane i & 31 (chunk i >> 5): the G positions a lane
// has in flight are 32 apart, each probe is one 32-byte T4Dir sector.  One funnel shift gives a k-mer
// code; the code of the previous position (for "equal to the previous k-mer", SeqSet.hpp:1376) comes from the
// neighbouring lane by shuffle.  Results per position: sw->cnt[i] (postings, bit 31 = taken), sw->lo[i].
// Returns true iff some list has >= 100 postings.  Loops over chunks are deliberately not fully unrolled: the kernel has
// to stay inside the instruction cache (a first, fully unrolled version over register arrays spent 8.7 of 16 stall
// cycles per issue on instruction fetch).
template <int G>
__device__ __forceinline__ bool t4p_probe_tile( const T4ProbeRead &R, T4ProbeWarp *sw, int tile0, int tileLen, int lane )
{
	bool large = false ;
	const int nChunks = ( tileLen + 31 ) >> 5 ;
	u64 carry = 0 ; // code of the last position of the previous chunk
	if ( tile0 > 0 )
	{
		int pass, q ;
		if ( t4p_active( R, tile0 - 1, pass, q ) )
			carry = t4p_extract( pass ? sw->rc : sw->fw, q, R.k ) ;
	}
#pragma unroll 1
	for ( int c0 = 0 ; c0 < nChunks ; c0 += G )
	{
		u64 key[G], v[G][4] ;
		u32 slot[G], tk[G] ;
#pragma unroll
		for ( int cc = 0 ; cc < G ; ++cc )
		{
			const int i = ( c0 + cc ) * 32 + lane ;
			int pass, q ;
			key[cc] = 0 ;
			slot[cc] = 0 ;
			tk[cc] = 0 ;
			if ( c0 + cc >= nChunks )
				continue ;                                       // warp-uniform
			const bool act = i < tileLen && t4p_active( R, tile0 + i, pass, q ) ;
			const u64 code = act ? t4p_extract( pass ? sw->rc : sw->fw, q, R.k ) : 0 ;
			u64 prev = __shfl_up_sync( 0xffffffffu, code, 1 ) ;
			if ( lane == 0 )
				prev = carry ;
			carry = __shfl_sync( 0xffffffffu, code, 31 ) ;
			if ( act )
			{
				if ( q == 0 || code != prev )
					tk[cc] = T4P_TAKEN ;
				// validity window: forward positions [q, q + k) or, for the reverse pass, [len - q - k, len - q)
				if ( !R.anyN || !t4p_has_n( sw->nm, pass ? R.len - q - R.k : q, R.k ) )
				{
					key[cc] = code + R.salt + 1 ;
					slot[cc] = (u32)( ( key[cc] * 0x9E3779B97F4A7C15ull ) >> 32 ) & R.dirMask ;
					t4p_ld256( R.dir + slot[cc], v[cc][0], v[cc][1], v[cc][2], v[cc][3] ) ;
				}
			}
		}
#pragma unroll
		for ( int cc = 0 ; cc < G ; ++cc )
		{
			const int i = ( c0 + cc ) * 32 + lane ;
			if ( c0 + cc >= nChunks )
				break ;
			u32 n = 0, l = 0 ;
			if ( key[cc] != 0 )
			{
				u64 kk = v[cc][0], lOff = v[cc][1], cw = v[cc][2], pad ;
				u32 s = slot[cc] ;
				while ( kk != key[cc] && kk != 0 ) // linear probing past a colliding slot
				{
					s = ( s + 1 ) & R.dirMask ;
					t4p_ld256( R.dir + s, kk, lOff, cw, pad ) ;
				}
				if ( kk == key[cc] )
				{
					n = (u32)cw ;
					l = (u32)( lOff >> 5 ) ;
					if ( n >= 100 )
						large = true ;
				}
			}
			if ( i < tileLen )
			{
				sw->cnt[i] = n | tk[cc] ;
				sw->lo[i] = l ;
			}
		}
	}
	__syncwarp() ;
	return __any_sync( 0xffffffffu, large ) ;
}

// No list reaches 100 postings: "taken" is the per-position predicate computed above (first k-mer of the pass, or code
// differs from the previous k-mer's -- N counted as A), and the hit slots are an exclusive prefix sum in position order.
// Here lane l owns the CONTIGUOUS positions [l * ppl, (l + 1) * ppl): a local sum, ONE warp scan, a local walk.
__device__ __forceinline__ void t4p_scan_fast( T4ProbeWarp *sw, int tileLen, int lane, T4ProbeScan &S )
{
	const int ppl = ( tileLen + 31 ) >> 5 ;
	const int i0 = lane * ppl, i1 = min( tileLen, i0 + ppl ) ;
	u32 local = 0, looks = 0 ;
#pragma unroll 1
	for ( int i = i0 ; i < i1 ; ++i )
	{
		const u32 cv = sw->cnt[i] ;
		if ( cv & T4P_TAKEN )
		{
			local += T4P_CNT( cv ) ;
			++looks ;
		}
	}
	u32 tot ;
	u32 o = S.total + t4p_warp_excl_scan( local, tot, lane ) ;
#pragma unroll 1
	for ( int i = i0 ; i < i1 ; ++i )
	{
		const u32 cv = sw->cnt[i] ;
		const bool emit = ( cv & T4P_TAKEN ) && T4P_CNT( cv ) > 0 ;
		sw->base[i] = emit ? o : T4P_NONE ;
		if ( emit )
			o += T4P_CNT( cv ) ;
	}
	S.total += tot ;
#pragma unroll
	for ( int d = 16 ; d > 0 ; d >>= 1 )
		looks += __shfl_xor_sync( 0xffffffffu, looks, d ) ;
	S.lookups += looks ;
	__syncwarp() ;
}

// Some list has >= 100 postings: the reference's loop, position by position; every lane runs the same scalar state machine
// over the sizes in shared memory (broadcast reads), lane 0 records the slots.
__device__ __forceinline__ void t4p_scan_serial( const T4ProbeRead &R, T4ProbeWarp *sw, int tile0, int tileLen, int lane, int allowTotalSkip,
	T4ProbeScan &S )
{
	const int skipLimit = R.k / 2 ;
	u64 code = 0 ;
	int lastX = -2 ;
#pragma unroll 1
	for ( int i = 0 ; i < tileLen ; ++i )
	{
		int pass, q ;
		u32 b = T4P_NONE ;
		if ( t4p_active( R, tile0 + i, pass, q ) )
		{
			if ( pass != S.curPass )
			{
				S.curPass = pass ;
				S.skipCnt = 0 ;
			}
			const u64 *W = pass ? sw->rc : sw->fw ;
			if ( q == 0 || lastX != tile0 + i - 1 )
				code = t4p_extract( W, q, R.k ) ;
			else
				code = ( ( code << 2 ) & R.mask ) | t4p_base_at( W, q + R.k - 1 ) ;
			lastX = tile0 + i ;
			const u32 size = T4P_CNT( sw->cnt[i] ) ;
			const int e = q + R.k - 1 ;
			bool setPrev = true ;
			if ( q == 0 || code != S.prev )
			{
				++S.lookups ;
				if ( size >= 100 && q != 0 && e != R.len - 1 && S.skipCnt < skipLimit )
				{
					++S.skipCnt ;
					setPrev = false ; // prevKmerCode keeps its stale value (SeqSet.hpp:1381-1388)
				}
				else if ( size >= 100 && allowTotalSkip )
					setPrev = false ;
				else
				{
					S.skipCnt = 0 ;
					if ( size > 0 )
					{
						b = S.total ;
						S.total += size ;
						if ( R.barcode == -1 && size > T4_BIG_REPEAT )
							S.big = 1 ;
					}
				}
			}
			if ( setPrev )
				S.prev = code ;
		}
		if ( lane == 0 )
			sw->base[i] = b ;
	}
	__syncwarp() ;
}

__device__ __forceinline__ u64 t4p_key( int pass, int q, u64 posting, int big )
{
	return t4_key_of( pass ? -1 : 1, (int)( posting >> 32 ), q, (int)(u32)posting, big ) ;
}

// Postings -> hit keys for one tile.  out: first key of this read.
template <int G>
__device__ __forceinline__ void t4p_emit_tile( const T4ProbeRead &R, T4ProbeWarp *sw, const char *A, int tile0, int tileLen, int lane,
	u64 *out, u32 &barPhase )
{
	const int nChunks = ( tileLen + 31 ) >> 5 ;
	// ---- lists of <= 4 postings: one sector, fetched by the owner lane (position i & 31 == lane); G lists in flight.
	// Hit slots grow with the position, so neighbouring lanes write neighbouring output ranges.
#pragma unroll 1
	for ( int c0 = 0 ; c0 < nChunks ; c0 += G )
	{
		u64 p[G][4] ;
		u32 n[G], b[G] ;
#pragma unroll
		for ( int cc = 0 ; cc < G ; ++cc )
		{
			const int i = ( c0 + cc ) * 32 + lane ;
			n[cc] = 0 ;
			if ( c0 + cc < nChunks && i < tileLen )
			{
				b[cc] = sw->base[i] ;
				const u32 cn = T4P_CNT( sw->cnt[i] ) ;
				if ( b[cc] != T4P_NONE && cn <= T4P_SHORT )
				{
					n[cc] = cn ;
					t4p_ld256( A + ( (u64)sw->lo[i] << 5 ), p[cc][0], p[cc][1], p[cc][2], p[cc][3] ) ;
				}
			}
		}
#pragma unroll
		for ( int cc = 0 ; cc < G ; ++cc )
			if ( n[cc] )
			{
				const int x = tile0 + ( c0 + cc ) * 32 + lane ;
				const int pass = x >= R.m ;
				const int q = pass ? x - R.m : x ;
				u64 *o = out + b[cc] ;
#pragma unroll
				for ( int j = 0 ; j < T4P_SHORT ; ++j )
					if ( j < (int)n[cc] )
						o[j] = t4p_key( pass, q, p[cc][j], 0 ) ;
			}
	}
	// ---- lists of 5 .. T4P_TMA_MAX postings: through the TMA staging tile.
	// (1) compact them, in position order, into a table in shared memory (sw->sb: position index per entry);
	// (2) rounds of up to 32 entries whose even-rounded lengths fit the tile: lane e owns entry w0 + e and issues its bulk
	//     copy, all wait on the mbarrier; (3) the staged slots are converted FLAT, 32 per step: every lane finds the list
	//     of its slot from the list heads inside the step's window (one REDUX.OR + popcount), so short lists do not idle lanes.
	u32 nLong = 0 ;
#pragma unroll 1
	for ( int c = 0 ; c < nChunks ; ++c )
	{
		const int i = c * 32 + lane ;
		const u32 cn = i < tileLen ? T4P_CNT( sw->cnt[i] ) : 0 ;
		const bool isLong = i < tileLen && cn > T4P_SHORT && cn <= T4P_TMA_MAX && sw->base[i] != T4P_NONE ;
		const u32 m = __ballot_sync( 0xffffffffu, isLong ) ;
		if ( isLong )
			sw->sb[nLong + __popc( m & ( ( 1u << lane ) - 1u ) )] = (u32)i ;
		nLong += __popc( m ) ;
	}
	__syncwarp() ;
#pragma unroll 1
	for ( u32 w0 = 0 ; w0 < nLong ; )
	{
		const u32 e = w0 + lane ;
		int pi = 0 ;
		u32 n = 0, v = 0 ;
		if ( e < nLong )
		{
			pi = (int)sw->sb[e] ;
			n = T4P_CNT( sw->cnt[pi] ) ;
			v = ( n + 1 ) & ~1u ;
		}
		u32 tot ;
		u32 so = t4p_warp_excl_scan( v, tot, lane ) ;
		const bool in = e < nLong && so + v <= T4P_STG ;                // a prefix of the 32 candidates (offsets are monotone)
		const int nIn = __popc( __ballot_sync( 0xffffffffu, in ) ) ;    // >= 1: a single list always fits (n <= T4P_TMA_MAX <= T4P_STG)
		const u32 slots = __shfl_sync( 0xffffffffu, so + v, nIn - 1 ) ;
		// the previous round's generic-proxy reads of the tile are ordered before the async-proxy writes of this one
		asm volatile( "fence.proxy.async.shared::cta;" ::: "memory" ) ;
		__syncwarp() ;
		if ( lane == 0 )
			t4p_bar_expect( &sw->bar, slots * 8 ) ;
		__syncwarp() ;
		if ( in )
			t4p_bulk_g2s( sw->stg + so, A + ( (u64)sw->lo[pi] << 5 ), v * 8, &sw->bar ) ;
		const u32 bo = in ? sw->base[pi] : 0 ;
		if ( !in )
			so = 0xffffffffu ;                                            // never "<= slot" in the search below
		t4p_bar_wait( &sw->bar, barPhase ) ;
		barPhase ^= 1 ;
		u32 passed = 0 ;                                                // lists that start before the current window
#pragma unroll 1
		for ( u32 s0 = 0 ; s0 < slots ; s0 += 32 )
		{
			const u32 sl = s0 + lane ;
			// list of slot sl = the last one starting at or before it: the round's lists are lanes 0 .. nIn-1 in staging
			// order, so one OR-reduction of "my list starts at window bit b" + a popcount replaces a search
			const u32 rel = so - s0 ;                                     // so = 0xffffffff (not staged) never lands in the window
			const u32 heads = __reduce_or_sync( 0xffffffffu, rel < 32u ? 1u << rel : 0u ) ;
			const int lo_ = (int)( passed + __popc( heads & ( 0xffffffffu >> ( 31 - lane ) ) ) ) - 1 ;
			passed += __popc( heads ) ;
			const u32 fn = __shfl_sync( 0xffffffffu, n, lo_ ) ;
			const u32 fso = __shfl_sync( 0xffffffffu, so, lo_ ) ;
			const u32 fbo = __shfl_sync( 0xffffffffu, bo, lo_ ) ;
			const int x = tile0 + __shfl_sync( 0xffffffffu, pi, lo_ ) ;
			const u32 j = sl - fso ;
			if ( sl < slots && j < fn )
			{
				const int pass = x >= R.m ;
				const int q = pass ? x - R.m : x ;
				out[fbo + j] = t4p_key( pass, q, sw->stg[sl], 0 ) ;
			}
		}
		w0 += nIn ;
		__syncwarp() ;
	}
	// ---- longer lists: streamed by the whole warp, two postings (128 bits) per lane and load
#pragma unroll 1
	for ( int c = 0 ; c < nChunks ; ++c )
	{
		const int i = c * 32 + lane ;
		u32 mask = __ballot_sync( 0xffffffffu, i < tileLen && sw->base[i] != T4P_NONE && T4P_CNT( sw->cnt[i] ) > T4P_TMA_MAX ) ;
		while ( mask )
		{
			const int src = __ffs( mask ) - 1 ;
			mask &= mask - 1 ;
			const int is = c * 32 + src ;
			const u32 n = T4P_CNT( sw->cnt[is] ), bo = sw->base[is] ;
			const char *l = A + ( (u64)sw->lo[is] << 5 ) ;
			const int x = tile0 + is ;
			const int pass = x >= R.m ;
			const int q = pass ? x - R.m : x ;
			const int big = ( R.barcode == -1 && n > T4_BIG_REPEAT ) ? 1 : 0 ;
			for ( u32 j = 2 * lane ; j < n ; j += 64 )
			{
				u64 a, b2 ;
				t4p_ld128( l + 8ull * j, a, b2 ) ;
				out[bo + j] = t4p_key( pass, q, a, big ) ;
				if ( j + 1 < n )
					out[bo + j + 1] = t4p_key( pass, q, b2, big ) ;
			}
		}
	}
}

// MINB: resident CTAs (= warps) per SM the register allocation is bounded for (24: 80 registers; 16: 128 registers)
template <int MINB, int G>
__global__ void __launch_bounds__( 32 * T4P_WARPS, MINB ) t4_probe_kernel( T4ProbeParams P )
{
	extern __shared__ __align__( 16 ) unsigned char t4p_dyn[] ; // T4P_WARPS x T4ProbeWarp (> 48 KB: dynamic, opted in by the host)
	const int lane = threadIdx.x & 31 ;
	T4ProbeWarp *sw = (T4ProbeWarp *)t4p_dyn + ( threadIdx.x >> 5 ) ;
	if ( lane == 0 )
		t4p_bar_init( &sw->bar ) ;
	__syncwarp() ;
	u32 barPhase = 0 ;
	u64 accLook = 0, accPost = 0, accBytes = 0, accUnsup = 0 ;
	while ( 1 )
	{
		unsigned long long w = 0 ;
		if ( lane == 0 )
			w = atomicAdd( (unsigned long long *)&P.ctrl[0], 1ull ) ;
		w = __shfl_sync( 0xffffffffu, w, 0 ) ;
		if ( (i64)w >= P.nReads )
			break ;
		const u64 ent = __ldg( P.ord + w ) ;
		const u32 ri = (u32)ent, si = (u32)( ent >> 32 ) ;
		const t4_read_desc *d = P.descs + ri ;
		const T4Stream *st = (const T4Stream *)( P.A + __ldg( P.streamOff + si ) ) ;
		T4ProbeRead R ;
		R.len = d->len ;
		R.barcode = d->barcode ;
		R.strand = d->strand_in ;
		R.k = st->kmerLength ;
		R.m = R.len - R.k + 1 ;
		R.nPos = 2 * R.m ;
		R.dir = (const T4Dir *)( P.A + st->dirOff ) ;
		R.dirMask = st->dirCap - 1 ;
		R.salt = st->considerBarcode ? ( (u64)( (u32)( R.barcode + 1 ) % T4_KINDEX_HASH_MAX ) << ( 2 * R.k ) ) : 0ull ;
		R.mask = ( 1ull << ( 2 * R.k ) ) - 1ull ; // k <= 31
		if ( R.len > T4_DEV_MAX_READ || R.len < R.k )
		{
			if ( lane == 0 )
			{
				P.hitOff[ri] = 0 ;
				P.hitCnt[ri] = 0 ;
				P.hitFlags[ri] = 0 ;
				if ( R.len > T4_DEV_MAX_READ )
					++accUnsup ;
			}
			continue ;
		}
		// packed read -> shared memory (<= 16 + 16 words + 16 mask words, zero padded)
		{
			const int W = (int)t4_pack_w( R.len ) ;
			const u64 *pk = P.packed + (u64)ri * P.packStride ;
			__syncwarp() ;
			if ( lane < 18 )
			{
				sw->fw[lane] = lane < W ? __ldg( pk + lane ) : 0 ;
				sw->rc[lane] = lane < W ? __ldg( pk + W + lane ) : 0 ;
			}
			u32 nmw = 0 ;
			if ( lane < 20 )
			{
				nmw = lane < W ? __ldg( (const u32 *)( pk + 2 * W ) + lane ) : 0 ;
				sw->nm[lane] = nmw ;
			}
			R.anyN = __any_sync( 0xffffffffu, nmw != 0 ) ;
			__syncwarp() ;
		}
		T4ProbeScan S ;
		const int nTiles = ( R.nPos + T4P_TILE - 1 ) / T4P_TILE ;
		u32 flags = 0 ;
		u64 *out = 0 ;
		u32 T = 0 ;
		// sweep 0 counts (directory probes + slot assignment), then the output range is reserved, sweep 1 emits.  A read
		// that fits one tile (<= 288 positions: 150 bp at k >= 7) keeps its probe results in shared memory between the
		// two; a longer one probes its tiles again (L1/L2 hits) and always uses the serial rules, which reduce to the
		// plain predicate when no list is large.
#pragma unroll 1
		for ( int sweep = 0 ; sweep < 2 ; ++sweep )
		{
			if ( sweep == 0 || nTiles > 1 )
			{
				S.prev = 0 ; S.skipCnt = 0 ; S.curPass = -1 ; S.total = 0 ; S.lookups = 0 ; S.big = 0 ;
			}
#pragma unroll 1
			for ( int t = 0 ; t < nTiles ; ++t )
			{
				const int tile0 = t * T4P_TILE ;
				const int tileLen = min( T4P_TILE, R.nPos - tile0 ) ;
				if ( sweep == 0 || nTiles > 1 )
				{
					const bool large = t4p_probe_tile<G>( R, sw, tile0, tileLen, lane ) ;
					if ( nTiles == 1 && !large )
						t4p_scan_fast( sw, tileLen, lane, S ) ;
					else
					{
						t4p_scan_serial( R, sw, tile0, tileLen, lane, P.allowTotalSkip, S ) ;
						flags |= 2 ;
					}
				}
				if ( sweep == 1 )
					t4p_emit_tile<G>( R, sw, P.A, tile0, tileLen, lane, out, barPhase ) ;
			}
			if ( sweep == 0 )
			{
				T = S.total ;
				unsigned long long o0 = 0 ;
				if ( lane == 0 )
					o0 = atomicAdd( (unsigned long long *)&P.ctrl[1], (unsigned long long)T ) ;
				o0 = __shfl_sync( 0xffffffffu, o0, 0 ) ;
				const bool fits = o0 + T <= P.keyCap ;
				if ( lane == 0 )
				{
					P.hitOff[ri] = o0 ;
					P.hitCnt[ri] = fits ? T : 0 ;
					P.hitFlags[ri] = flags | ( S.big ? 1u : 0u ) ;
					if ( !fits )
						P.ctrl[2] = 1 ;
				}
				accLook += S.lookups ;
				accPost += T ;
				accBytes += ( R.len + 3 ) / 4 ;
				if ( !fits || T == 0 )
					break ;
				out = P.keys + o0 ;
			}
		}
		// barcode filter (SeqSet.hpp:1418): hits on contigs of another barcode become invalid keys.  Off the hot path: only
		// reads that carry a barcode pay for it, in one pass over their own keys.
		if ( R.barcode != -1 && out != 0 )
		{
			const T4Contig *seqs = (const T4Contig *)( P.A + st->seqsOff ) ;
			__syncwarp() ;
			for ( u32 t = lane ; t < T ; t += 32 )
			{
				const u64 key = __ldcg( out + t ) ;
				if ( __ldg( &seqs[t4_key_idx( key )].barcode ) != R.barcode )
					out[t] = T4_KEY_INVALID ;
			}
		}
	}
	if ( lane == 0 )
	{
		if ( accLook ) atomicAdd( (unsigned long long *)&P.ctrl[3], (unsigned long long)accLook ) ;
		if ( accPost )
		{
			atomicAdd( (unsigned long long *)&P.ctrl[4], (unsigned long long)accPost ) ;
			atomicAdd( (unsigned long long *)&P.ctrl[5], (unsigned long long)accPost ) ;
		}
		if ( accBytes ) atomicAdd( (unsigned long long *)&P.ctrl[6], (unsigned long long)accBytes ) ;
		if ( accUnsup ) atomicAdd( (unsigned long long *)&P.ctrl[7], (unsigned long long)accUnsup ) ;
	}
}

// Visit order of the probe: reads of one set together, inside a set by length bucket (32 bases per bucket, longest
// first) so that the warps of a CTA carry equal numbers of k-mers.  One CTA per set.
__global__ void t4_bucket_kernel( const t4_read_desc *descs, const i64 *descOff, u64 *ord )
{
	__shared__ u32 hist[17], cur[17] ;
	const int s = blockIdx.x ;
	const i64 lo = descOff[s], hi = descOff[s + 1] ;
	if ( threadIdx.x < 17 )
		hist[threadIdx.x] = 0 ;
	__syncthreads() ;
	for ( i64 i = lo + threadIdx.x ; i < hi ; i += blockDim.x )
	{
		int b = 16 - min( 16, max( 0, descs[i].len ) >> 5 ) ;
		atomicAdd( &hist[b], 1u ) ;
	}
	__syncthreads() ;
	if ( threadIdx.x == 0 )
	{
		u32 a = 0 ;
		for ( int b = 0 ; b < 17 ; ++b )
		{
			cur[b] = a ;
			a += hist[b] ;
		}
	}
	__syncthreads() ;
	for ( i64 i = lo + threadIdx.x ; i < hi ; i += blockDim.x )
	{
		int b = 16 - min( 16, max( 0, descs[i].len ) >> 5 ) ;
		u32 p = atomicAdd( &cur[b], 1u ) ;
		ord[lo + p] = (u64)(u32)i | ( (u64)(u32)s << 32 ) ;
	}
}

#endif // T4_CUDA
#endif
