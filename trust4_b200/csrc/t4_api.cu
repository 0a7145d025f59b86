// C ABI of include/trust4_b200.h over the stream engine (t4_engine.h).
//
// Product build: nvcc -gencode arch=compute_90a,code=sm_90a -> libtrust4_b200.so.  The hot path runs
// only on the GPU; every entry point fails with T4_E_NODEVICE when no device is present.
// Test-only emulation build (tests/emu, g++ -x c++ -DT4_EMU -DT4_PREFIX=t4emu_): the same host logic with
// the "device" being host memory and one emulated thread per stream; it exports t4emu_* symbols only.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <limits.h>
#include <vector>
#include <map>
#include <string>
#include <mutex>
#include <thread>

#include "t4_engine.h"
#include "t4_assign.h"
#include "t4_refscan.h"
#include "t4_annot.h"
#include "t4_kcount.h"
#include "t4_readsort.h"

#if T4_CUDA
#include <cuda_runtime.h>
#include "t4_probe.cuh"
#endif
#include "t4_shard.h"

#ifdef T4_EMU
#define T4_CAT2( a, b ) a##b
#define T4_CAT( a, b ) T4_CAT2( a, b )
#define T4_API( name ) T4_CAT( t4emu_, name )
#else
#define T4_API( name ) t4_##name
#endif

// ---------------------------------------------------------------------------
// backend
// ---------------------------------------------------------------------------
static std::string g_err ;
static void set_err( const std::string &s ) { g_err = s ; }

#define T4_MIN_BLOCKS 4 // resident CTAs per SM the op kernels are register-bounded for

#if T4_CUDA
#define CK( call )                                                                 \
	do                                                                             \
	{                                                                              \
		cudaError_t e_ = ( call ) ;                                                \
		if ( e_ != cudaSuccess )                                                   \
		{                                                                          \
			set_err( std::string( #call ) + ": " + cudaGetErrorString( e_ ) ) ;    \
			return T4_E_CUDA ;                                                     \
		}                                                                          \
	} while ( 0 )

// The kernels are thin wrappers: their bodies are device functions the emulation runs too (see the launchers below).
__global__ void __launch_bounds__( T4_MAX_NT, T4_MIN_BLOCKS ) t4_stream_kernel( char *A, T4Op *ops, const int *gapTable )
{
	__shared__ T4Smem sm ;
	T4Ctx cx = t4_ctx( A, ops[blockIdx.x].streamOff, &sm, threadIdx.x, blockDim.x ) ;
	c_run_op( cx, ops + blockIdx.x, gapTable ) ;
}

// The read-only passes over finished sets (t4_assign.h) are a kernel of their own: they share the engine's collectives
// but must not weigh on the register allocation of the assembly loop above.
__global__ void __launch_bounds__( T4_MAX_NT, T4_MIN_BLOCKS ) t4_aux_kernel( char *A, T4Op *ops )
{
	__shared__ T4Smem sm ;
	T4Ctx cx = t4_ctx( A, ops[blockIdx.x].streamOff, &sm, threadIdx.x, blockDim.x ) ;
	c_run_aux_op( cx, ops + blockIdx.x ) ;
}

// GetOverlapsFromRead and AnnotateRead on a reference gene set (t4_annot.h): a kernel of its own, so that the other op
// kernels keep their exact SASS
__global__ void __launch_bounds__( T4_MAX_NT, T4_MIN_BLOCKS ) t4_annot_kernel( char *A, T4Op *ops )
{
	__shared__ T4Smem sm ;
	T4Ctx cx = t4_ctx( A, ops[blockIdx.x].streamOff, &sm, threadIdx.x, blockDim.x ) ;
	c_run_annot_op( cx, ops + blockIdx.x ) ;
}

// one merge pass of the read sort (t4_readsort.h)
__global__ void t4_readsort_kernel( T4SortParams P )
{
	for ( i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x ; i < P.n ; i += (i64)gridDim.x * blockDim.x )
		t4_sort_merge_one<T4SortRec>( P, i ) ;
}

// the same pass in the --barcode order (CompReadWithBarcode)
__global__ void t4_readsort_bc_kernel( T4SortParams P )
{
	for ( i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x ; i < P.n ; i += (i64)gridDim.x * blockDim.x )
		t4_sort_merge_one<T4SortRecBc>( P, i ) ;
}

__global__ void t4_mate_overlap_kernel( T4MateParams P )
{
	for ( i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x ; i < P.n ; i += (i64)gridDim.x * blockDim.x )
		t4_mate_overlap_one( P, i ) ;
}

__global__ void t4_pack_reads_kernel( T4PackReadsParams P )
{
	for ( i64 g = (i64)blockIdx.x * blockDim.x + threadIdx.x ; g < P.n * P.wMax ; g += (i64)gridDim.x * blockDim.x )
		t4_pack_read_word( P, g ) ;
}

__global__ void t4_dp_kernel( T4DpParams P )
{
	for ( int i = blockIdx.x * blockDim.x + threadIdx.x ; i < P.n ; i += gridDim.x * blockDim.x )
		t4_dp_one( P, i ) ;
}

// k-mer counting / per-read count statistics (t4_kcount.h): persistent warps, batches of reads handed out by an atomic cursor
__global__ void __launch_bounds__( T4_MAX_NT ) t4_kcount_kernel( T4KcParams P, int stats )
{
	__shared__ T4KcSmem sm[T4_MAX_NT / T4_KC_GROUP] ;
	T4KcCtx cx ;
	cx.sm = &sm[threadIdx.x / T4_KC_GROUP] ;
	cx.tid = threadIdx.x % T4_KC_GROUP ;
	cx.nt = T4_KC_GROUP ;
	const T4KcBarcode B = { 0, 0, 0 } ;
	if ( stats )
		kc_stats_body<false>( cx, P, B ) ;
	else
		kc_count_body<false>( cx, P, B ) ;
}

// the per-cell pass: one table keyed by (barcode, k-mer) for the barcodes of [B.lo, B.lo + 2^21)
__global__ void __launch_bounds__( T4_MAX_NT ) t4_kcount_bc_kernel( T4KcParams P, int stats, T4KcBarcode B )
{
	__shared__ T4KcSmem sm[T4_MAX_NT / T4_KC_GROUP] ;
	T4KcCtx cx ;
	cx.sm = &sm[threadIdx.x / T4_KC_GROUP] ;
	cx.tid = threadIdx.x % T4_KC_GROUP ;
	cx.nt = T4_KC_GROUP ;
	if ( stats )
		kc_stats_body<true>( cx, P, B ) ;
	else
		kc_count_body<true>( cx, P, B ) ;
}

__global__ void t4_init_kernel( char *A, u64 base, T4InitParams ip )
{
	c_init_block( A, base, ip, blockIdx.x, threadIdx.x, blockDim.x ) ;
}

__global__ void t4_gather_kernel( char *A, const T4Contig *ct, const u64 *outOff, char *out, int n )
{
	t4_gather_block( A, ct, outOff, out, n, blockIdx.x, threadIdx.x, blockDim.x ) ;
}

__global__ void t4_pack_size_kernel( char *A, const u64 *streamOff, u64 *sizes, u64 *counts )
{
	t4_pack_size_block( A, streamOff, sizes, counts, blockIdx.x, threadIdx.x, blockDim.x ) ;
}

__global__ void t4_pack_kernel( char *A, const u64 *streamOff, const u64 *outOff, char *out )
{
	t4_pack_block( A, streamOff, outOff, out, blockIdx.x, threadIdx.x, blockDim.x ) ;
}

// Test entry for the two DP routines the stream kernel really runs (equal lengths: overhangs and same-diagonal gaps):
// variant 0 = t4_dp_equal (register-resident banded DP, one thread per problem, ExtendOverlap),
// variant 1 = w_stage_side + w_dp_equal_half (half-warp anti-diagonal DP over staged IsBaseEqual nibbles, gap scoring;
//             it has no fast path: the caller only runs it when the diagonal has > 2 mismatches),
// variant 2 = w_side_pair (ExtendOverlap's overhang pass: problems 2k and 2k+1 on the two halves of warp k, as a left
//             side, scanned from its end, and a right side); writes each problem's T4SideStats, not its edit string.
// One warp per problem (variant 2: per pair).  scratch: per problem 13 * actStride u32 traceback words + an edit-string
// buffer (large n).  The problems come as posWeight columns; the kernel derives their equality bytes (t4_eq) itself.
__global__ void t4_dp_hot_kernel( int n, int variant, const int *tw, const i64 *off, const char *p, signed char *align, const i64 *alignOff,
	int *score, u32 *scratch, const i64 *scratchOff )
{
	__shared__ unsigned char eqb[2][T4_DEV_MAX_READ] ;
	__shared__ u32 nib[2][64] ;
	__shared__ u32 bits[2][16] ;
	__shared__ u32 act[2][13 * T4_WACT_WORDS] ;
	__shared__ signed char wal[2][2 * 16 * T4_WACT_WORDS + 8] ;
	if ( variant == 2 )
	{
		T4Ctx cx ;
		cx.tid = threadIdx.x ;
		cx.nt = 32 ;
		T4DpSide s[2] ;
		for ( int h = 0 ; h < 2 ; ++h )
		{
			const int k = 2 * blockIdx.x + h ;
			T4DpSide &d = s[h] ;
			d.n = ( k < n ) ? (int)( off[k + 1] - off[k] ) : 0 ;
			for ( int t = threadIdx.x ; t < d.n ; t += 32 )
				eqb[h][t] = (unsigned char)t4_eq_nibble( tw + 4 * ( off[k] + t ) ) ;
			d.te = eqb[h] ;
			d.p = p + off[k < n ? k : 0] ;
			d.fromEnd = ( h == 0 ) ;
			const bool small = d.n < 16 * T4_WACT_WORDS ;
			d.actStride = small ? T4_WACT_WORDS : ( d.n / 16 + 2 ) ;
			d.act = small ? act[h] : scratch + scratchOff[k] ;
			d.alCap = small ? (int)sizeof( wal[0] ) : 2 * d.n + 8 ;
			d.al = small ? wal[h] : (signed char *)( scratch + scratchOff[k] + 13 * d.actStride ) ;
		}
		__syncwarp() ;
		T4SideStats r[2] ;
		w_side_pair( cx, s[0], s[1], nib, bits, r[0], r[1] ) ;
		for ( int h = 0 ; h < 2 ; ++h )
		{
			const int k = 2 * blockIdx.x + h ;
			if ( threadIdx.x == 0 && k < n )
			{
				int *o = (int *)( align + alignOff[k] ) ;
				o[0] = r[h].m ;
				o[1] = r[h].x ;
				o[2] = r[h].ind ;
				o[3] = r[h].good ;
			}
		}
		return ;
	}
	int i = blockIdx.x ;
	if ( i >= n )
		return ;
	const int len = (int)( off[i + 1] - off[i] ) ;
	const int lane = threadIdx.x ;
	const int *t = tw + 4 * off[i] ;
	const char *pp = p + off[i] ;
	signed char *out = align + alignOff[i] ;
	if ( variant == 0 )
	{
		if ( lane == 0 )
			score[i] = t4_dp_equal( t, pp, len, out, scratch + scratchOff[i], false, 0 ) ;
		return ;
	}
	T4Ctx cx ;
	cx.tid = lane ;
	cx.nt = 32 ;
	for ( int x = lane ; x < len ; x += 32 )
		eqb[0][x] = (unsigned char)t4_eq_nibble( t + 4 * x ) ;
	__syncwarp() ;
	int matches = w_stage_side( eqb[0], pp, len, nib[0], bits[0], lane ) ;
	(void)matches ;
	const bool small = len < 16 * T4_WACT_WORDS ;
	const int actStride = small ? T4_WACT_WORDS : ( len / 16 + 2 ) ;
	u32 *actBase = small ? act[lane < 16 ? 0 : 1] : scratch + scratchOff[i] + ( lane < 16 ? 0 : 13 * actStride ) ;
	const int acap = small ? (int)sizeof( wal[0] ) : 2 * len + 8 ;
	signed char *abuf = small ? wal[lane < 16 ? 0 : 1] : (signed char *)( scratch + scratchOff[i] + 26 * actStride ) + ( lane < 16 ? 0 : acap ) ;
	int alen = 0 ;
	int sc = w_dp_equal_half( cx, nib[0], pp, lane < 16 ? len : 0, abuf, acap, &alen, actBase, actStride ) ;
	alen = __shfl_sync( 0xffffffffu, alen, 0 ) ;
	sc = __shfl_sync( 0xffffffffu, sc, 0 ) ;
	signed char *buf0 = small ? wal[0] : (signed char *)( scratch + scratchOff[i] + 26 * actStride ) ;
	for ( int x = lane ; x <= alen ; x += 32 )
		out[x] = ( x == alen ) ? (signed char)-1 : buf0[acap - 1 - alen + x] ;
	if ( lane == 0 )
		score[i] = sc ;
}
#else
#define CK( call ) do { } while ( 0 )
#endif

struct Engine
{
	bool up ;
	int device ;
	int sms ;          // SM count of the device
	char *A ;          // arena base (device or, in the emulation, host)
	size_t cap ;
	int nt ;
	int *gapTable ;    // device int[40]
	int hostGap[40] ;
	// staging (device)
	char *stage ;
	size_t stageCap ;
	// grow-only device buffer reused by t4_streams_run for the uploaded workload (no cudaMalloc per call)
	char *wl ;
	size_t wlCap ;
	Engine() : up( false ), device( 0 ), sms( 0 ), A( 0 ), cap( 0 ), nt( 128 ), gapTable( 0 ), stage( 0 ), stageCap( 0 ), wl( 0 ), wlCap( 0 ) {}
} ;
static Engine E ;
static std::mutex g_mu ;

// workers of the read-only passes (one scratch stream each): one resident wave of the auxiliary kernels
static int resident_workers() { return T4_CUDA ? E.sms * T4_MIN_BLOCKS : 2 ; }

static int dmalloc( void **p, size_t n )
{
#if T4_CUDA
	CK( cudaMalloc( p, n ) ) ;
#else
	*p = malloc( n ) ;
	if ( !*p ) return T4_E_NOMEM ;
#endif
	return 0 ;
}
static void dfree( void *p )
{
#if T4_CUDA
	cudaFree( p ) ;
#else
	free( p ) ;
#endif
}
static int h2d( void *d, const void *h, size_t n )
{
	if ( n == 0 ) return 0 ;
#if T4_CUDA
	CK( cudaMemcpy( d, h, n, cudaMemcpyHostToDevice ) ) ;
#else
	memcpy( d, h, n ) ;
#endif
	return 0 ;
}
// ordered on `stream`; the host buffer may be reused when it returns
static int h2d_async( void *d, const void *h, size_t n, void *stream )
{
#if T4_CUDA
	CK( cudaMemcpyAsync( d, h, n, cudaMemcpyHostToDevice, (cudaStream_t)stream ) ) ;
#else
	memcpy( d, h, n ) ;
#endif
	return 0 ;
}
static int d2h( void *h, const void *d, size_t n )
{
	if ( n == 0 ) return 0 ;
#if T4_CUDA
	CK( cudaMemcpy( h, d, n, cudaMemcpyDeviceToHost ) ) ;
#else
	memcpy( h, d, n ) ;
#endif
	return 0 ;
}
static int dzero( void *d, size_t n, void *stream = 0 )
{
#if T4_CUDA
	CK( cudaMemsetAsync( d, 0, n, (cudaStream_t)stream ) ) ;
#else
	memset( d, 0, n ) ;
#endif
	return 0 ;
}
static int dsync()
{
#if T4_CUDA
	CK( cudaDeviceSynchronize() ) ;
#endif
	return 0 ;
}

// One device allocation carved into parts in the order they are added, each 256-byte aligned.  add() names the pointer
// a part goes to; alloc() makes the allocation and sets the pointers (place() sets them into a buffer the caller owns).
// The allocation is freed when the DevBuf goes out of scope unless keep() hands it over.
namespace {
struct DevBuf
{
	struct Part { size_t off ; void *ptr ; void ( *set )( void *ptr, char *at ) ; } ;
	std::vector<Part> parts ;
	size_t bytes = 0 ;
	char *base = 0 ;
	bool owned = false ;
	template <class T> void add( T *&p, size_t n )
	{
		parts.push_back( { bytes, &p, []( void *ptr, char *at ) { *(T **)ptr = (T *)at ; } } ) ;
		bytes += ( n + 255 ) & ~(size_t)255 ;
	}
	void place( char *at )
	{
		base = at ;
		for ( const Part &x : parts )
			x.set( x.ptr, at + x.off ) ;
	}
	int alloc()
	{
		void *p = 0 ;
		int r = dmalloc( &p, bytes ) ;
		if ( r ) return r ;
		place( (char *)p ) ;
		owned = true ;
		return 0 ;
	}
	char *keep() { owned = false ; return base ; }
	~DevBuf() { if ( owned ) dfree( base ) ; }
} ;
}

// ---- launchers: the kernel on the device; in the emulation its device body, in order, on one thread (tid 0, nt 1) ----
enum { T4K_STREAM, T4K_AUX, T4K_ANNOT } ;

// one CTA of E.nt threads per op record, of the stream, auxiliary or annotation kernel
static int launch_ops( int kernel, T4Op *dOps, int n, void *stream )
{
#if T4_CUDA
	cudaStream_t cs = (cudaStream_t)stream ;
	if ( kernel == T4K_STREAM )
		t4_stream_kernel<<<n, E.nt, 0, cs>>>( E.A, dOps, E.gapTable ) ;
	else if ( kernel == T4K_AUX )
		t4_aux_kernel<<<n, E.nt, 0, cs>>>( E.A, dOps ) ;
	else
		t4_annot_kernel<<<n, E.nt, 0, cs>>>( E.A, dOps ) ;
	CK( cudaGetLastError() ) ;
#else
	(void)stream ;
	T4Smem *sm = new T4Smem ;
	for ( int b = 0 ; b < n ; ++b )
	{
		T4Ctx cx = t4_ctx( E.A, dOps[b].streamOff, sm, 0, 1 ) ;
		if ( kernel == T4K_STREAM )
			c_run_op( cx, dOps + b, E.gapTable ) ;
		else if ( kernel == T4K_AUX )
			c_run_aux_op( cx, dOps + b ) ;
		else
			c_run_annot_op( cx, dOps + b ) ;
	}
	delete sm ;
#endif
	return 0 ;
}

// The kernel argument of launch_blocks / launch_items: the kernel on the device, its device body in the emulation.
#if T4_CUDA
#define T4_KERNEL( kernel, body ) kernel
#else
#define T4_KERNEL( kernel, body ) body
#endif

// grid CTAs of `threads` threads; the emulation runs body( args..., b, 0, 1 ) for every block b
template <class K, class... A> static int launch_blocks( K kernel, int grid, int threads, A... args )
{
#if T4_CUDA
	kernel<<<grid, threads>>>( args... ) ;
	CK( cudaGetLastError() ) ;
#else
	(void)threads ;
	for ( int b = 0 ; b < grid ; ++b )
		kernel( args..., b, 0, 1 ) ;
#endif
	return 0 ;
}

// one thread per item i < n (n > 0), a grid-stride loop over at most 16 CTAs per SM; the emulation runs body( p, i )
template <class K, class P> static int launch_items( K kernel, const P &p, i64 n, int threads )
{
#if T4_CUDA
	i64 blocks = ( n + threads - 1 ) / threads ;
	if ( blocks > (i64)E.sms * 16 )
		blocks = (i64)E.sms * 16 ;
	kernel<<<(int)blocks, threads>>>( p ) ;
	CK( cudaGetLastError() ) ;
#else
	(void)threads ;
	for ( i64 i = 0 ; i < n ; ++i )
		kernel( p, i ) ;
#endif
	return 0 ;
}

// SeqSet::ComputeNomatchGapLimit (SeqSet.hpp:2476-2482): host pow/log, like the reference
static int nomatch_gap_limit( int kl )
{
	double readAccuracy = 0.8 ;
	double kmerHitProb = pow( readAccuracy, kl ) ;
	int ret = int( kl * ( log( 0.01 ) / log( 1 - kmerHitProb ) ) ) + 1 ;
	return ret ;
}

static int ensure_stage( size_t n )
{
	if ( n <= E.stageCap )
		return 0 ;
	if ( E.stage )
		dfree( E.stage ) ;
	size_t c = E.stageCap ? E.stageCap : ( 1 << 20 ) ;
	while ( c < n )
		c *= 2 ;
	void *p = 0 ;
	int r = dmalloc( &p, c ) ;
	if ( r )
	{
		E.stage = 0 ;
		E.stageCap = 0 ;
		return r ;
	}
	E.stage = (char *)p ;
	E.stageCap = c ;
	return 0 ;
}

// host-side bump allocation (only between launches)
static int arena_alloc( size_t bytes, u64 *off )
{
	T4Global g ;
	int r = d2h( &g, E.A, sizeof( u64 ) * 2 ) ;
	if ( r ) return r ;
	bytes = ( bytes + 255 ) & ~(size_t)255 ;
	u64 top = ( g.top + 255 ) & ~255ull ;
	if ( top + bytes > g.cap )
	{
		set_err( "device arena exhausted" ) ;
		return T4_E_NOMEM ;
	}
	*off = top ;
	top += bytes ;
	return h2d( E.A, &top, sizeof( u64 ) ) ;
}

struct t4_seqset
{
	u64 off ;
	int k ;
	bool alive ;
	uint32_t gen ;
} ;
static uint32_t g_gen = 1 ;

struct t4_workload
{
	char *buf ;            // one device allocation
	size_t bytes ;
	i64 nDescs ;
	size_t poolBytes ;
	int nNames ;
	// device pointers into buf
	t4_read_desc *descs ;
	char *pool ;
	T4Names *names ;
	int32_t *ret ;
	int8_t *strands ;
	int32_t *rescue ;
	int32_t *rescueList ;
	int8_t *good ;
	int32_t *info ;
	uint8_t *events ;
	T4Op *ops ;
	int opCap ;
	bool persistent ;
	u64 *packed ;          // 2-bit packed reads, record i at packed + i * packStride (t4_common.h)
	u64 packStride ;
	bool usePacked ;       // every read is pure ACGTN: the stream kernel assembles from the packed pool
	bool ran ;             // the result arrays hold the outcome of an assembly run (t4_streams_run_resident)
} ;

extern "C" {

const char *T4_API( last_error )( void ) { return g_err.c_str() ; }
const char *T4_API( version )( void )
{
	return T4_CUDA ? "trust4_b200 0.1.0 (sm_90a)" : "trust4_b200 0.1.0 (TEST EMULATION - not a product build)" ;
}

int T4_API( shutdown )( void )
{
	std::lock_guard<std::mutex> lk( g_mu ) ;
	if ( !E.up )
		return 0 ;
	dsync() ;
	dfree( E.A ) ;
	if ( E.gapTable )
		dfree( E.gapTable ) ;
	if ( E.stage )
		dfree( E.stage ) ;
	if ( E.wl )
		dfree( E.wl ) ;
	E = Engine() ;
	++g_gen ;
	return 0 ;
}

int T4_API( init )( int device, size_t arena_bytes )
{
	std::lock_guard<std::mutex> lk( g_mu ) ;
	if ( E.up )
		return 0 ;
#if T4_CUDA
	int nd = 0 ;
	if ( cudaGetDeviceCount( &nd ) != cudaSuccess || nd == 0 )
	{
		set_err( "no CUDA device: trust4_b200 has no CPU fallback" ) ;
		return T4_E_NODEVICE ;
	}
	if ( device < 0 )
		CK( cudaGetDevice( &device ) ) ;
	CK( cudaSetDevice( device ) ) ;
	CK( cudaDeviceGetAttribute( &E.sms, cudaDevAttrMultiProcessorCount, device ) ) ;
	if ( arena_bytes == 0 )
	{
		size_t fr = 0, tot = 0 ;
		CK( cudaMemGetInfo( &fr, &tot ) ) ;
		arena_bytes = fr / 2 ;
	}
#else
	if ( arena_bytes == 0 )
		arena_bytes = 1ull << 30 ;
#endif
	const char *env = getenv( "T4_ARENA_MB" ) ;
	if ( env )
		arena_bytes = (size_t)atoll( env ) << 20 ;
	env = getenv( "T4_NT" ) ;
	if ( env )
		E.nt = atoi( env ) ;
#if T4_CUDA
	// the warp-collective sections (ballots with a full mask, per-warp shared arrays) need whole warps
	if ( E.nt < 32 || E.nt > T4_MAX_NT || ( E.nt & ( E.nt - 1 ) ) )
	{
		set_err( "T4_NT must be 32, 64 or 128" ) ;
		E.nt = 128 ;
		return T4_E_INVAL ;
	}
#else
	E.nt = 1 ;
#endif
	void *p = 0 ;
	int r = dmalloc( &p, arena_bytes ) ;
	if ( r )
		return r ;
	E.A = (char *)p ;
	E.cap = arena_bytes ;
	E.device = device ;
	T4Global g ;
	memset( &g, 0, sizeof( g ) ) ;
	g.top = ( sizeof( T4Global ) + 255 ) & ~255ull ;
	g.cap = arena_bytes ;
	r = h2d( E.A, &g, sizeof( g ) ) ;
	for ( int k = 0 ; k < 40 ; ++k )
		E.hostGap[k] = ( k >= 2 && k <= 32 ) ? nomatch_gap_limit( k ) : 0 ;
	p = 0 ;
	if ( !r )
		r = dmalloc( &p, sizeof( E.hostGap ) ) ;
	E.gapTable = (int *)p ;
	if ( !r )
		r = h2d( E.gapTable, E.hostGap, sizeof( E.hostGap ) ) ;
	if ( r )
	{
		// a failed init leaves nothing behind: the next t4_init() starts from scratch
		if ( E.gapTable )
			dfree( E.gapTable ) ;
		dfree( E.A ) ;
		E.gapTable = 0 ;
		E.A = 0 ;
		E.cap = 0 ;
		return r ;
	}
	E.up = true ;
	return 0 ;
}

static int ensure_up()
{
	if ( E.up )
		return 0 ;
	return T4_API( init )( -1, 0 ) ;
}

// Release every seqset and workload-independent allocation of the arena (all t4_seqset handles die).
int T4_API( reset )( void )
{
	if ( !E.up )
		return 0 ;
	int r = dsync() ;
	if ( r ) return r ;
	T4Global g ;
	memset( &g, 0, sizeof( g ) ) ;
	g.top = ( sizeof( T4Global ) + 255 ) & ~255ull ;
	g.cap = E.cap ;
	++g_gen ;
	return h2d( E.A, &g, sizeof( g ) ) ;
}

int T4_API( arena_stats )( size_t *used, size_t *capacity )
{
	if ( !E.up )
		return T4_E_INVAL ;
	T4Global g ;
	int r = d2h( &g, E.A, 16 ) ;
	if ( r ) return r ;
	if ( used ) *used = g.top ;
	if ( capacity ) *capacity = g.cap ;
	return 0 ;
}

int T4_API( last_counters )( uint64_t *c )
{
	if ( !E.up )
		return T4_E_INVAL ;
	T4Global g ;
	int r = d2h( &g, E.A, sizeof( g ) ) ;
	if ( r ) return r ;
	memcpy( c, g.counters, sizeof( g.counters ) ) ;
	return 0 ;
}

// Create n seqsets in one go (one init launch).  handles[i] receives the new set.
static int seqsets_create_impl( int n, int kmer_length, int hit_len_required, int consider_barcode, t4_seqset **handles ) ;

int T4_API( seqsets_create )( int n, int kmer_length, t4_seqset **handles )
{
	return seqsets_create_impl( n, kmer_length, 31, 0, handles ) ;
}

// The same with SetHitLenRequired / SetConsiderBarcodeInIndexHash applied to every set by the init launch
// (main.cpp:1549-1565 configures the set once before the loop; thousands of streams should not cost thousands of copies).
int T4_API( seqsets_create_ex )( int n, int kmer_length, int hit_len_required, int consider_barcode, t4_seqset **handles )
{
	if ( consider_barcode && kmer_length > 15 )
	{
		set_err( "barcode-salted index needs k <= 15" ) ;
		return T4_E_UNSUPPORTED ;
	}
	return seqsets_create_impl( n, kmer_length, hit_len_required, consider_barcode ? 1 : 0, handles ) ;
}

static int seqsets_create_impl( int n, int kmer_length, int hit_len_required, int consider_barcode, t4_seqset **handles )
{
	int r = ensure_up() ;
	if ( r ) return r ;
	if ( n <= 0 || kmer_length < 2 || kmer_length > 31 )
	{
		set_err( "bad k-mer length / count" ) ;
		return T4_E_INVAL ;
	}
	T4InitParams ip ;
	ip.hitLenRequired = hit_len_required ;
	ip.considerBarcode = consider_barcode ;
	ip.kmerLength = kmer_length ;
	ip.nomatchGapLimit = E.hostGap[kmer_length] ;
	ip.nThreads = E.nt ;
	ip.seqCap = 64 ;
	ip.dirCap = 2048 ;
	ip.hitCap = 2048 ;
	ip.ovlCap = 64 ;
	ip.footprint = 0 ;
	u64 fp = ( t4_stream_footprint( ip ) + 255 ) & ~255ull ;
	ip.footprint = (u32)fp ;
	u64 base ;
	r = arena_alloc( fp * n, &base ) ;
	if ( !r ) r = launch_blocks( T4_KERNEL( t4_init_kernel, c_init_block ), n, 128, E.A, base, ip ) ;
	if ( !r ) r = dsync() ;
	if ( r ) return r ;
	for ( int i = 0 ; i < n ; ++i )
	{
		t4_seqset *s = new t4_seqset ;
		s->off = base + (u64)i * fp ;
		s->k = kmer_length ;
		s->alive = true ;
		s->gen = g_gen ;
		handles[i] = s ;
	}
	return 0 ;
}

t4_seqset *T4_API( seqset_create )( int kmer_length )
{
	t4_seqset *s = 0 ;
	if ( T4_API( seqsets_create )( 1, kmer_length, &s ) )
		return 0 ;
	return s ;
}

void T4_API( seqset_destroy )( t4_seqset *s )
{
	// arena memory is reclaimed by t4_reset() / t4_shutdown() (bump allocator)
	delete s ;
}

static int check( t4_seqset *s )
{
	if ( !s || !E.up || s->gen != g_gen )
	{
		set_err( "stale or null seqset handle" ) ;
		return T4_E_INVAL ;
	}
	return 0 ;
}

static int get_stream( t4_seqset *s, T4Stream *st )
{
	int r = check( s ) ;
	if ( r ) return r ;
	return d2h( st, E.A + s->off, sizeof( T4Stream ) ) ;
}

static int put_field( t4_seqset *s, size_t fieldOff, const void *v, size_t n )
{
	int r = check( s ) ;
	if ( r ) return r ;
	return h2d( E.A + s->off + fieldOff, v, n ) ;
}

int T4_API( seqset_set_hit_len_required )( t4_seqset *s, int l ) { return put_field( s, offsetof( T4Stream, hitLenRequired ), &l, sizeof( int ) ) ; }
int T4_API( seqset_set_novel_seq_similarity )( t4_seqset *s, double v ) { return put_field( s, offsetof( T4Stream, novelSeqSimilarity ), &v, sizeof( double ) ) ; }
int T4_API( seqset_set_consider_barcode_in_hash )( t4_seqset *s, int on )
{
	int v = on ? 1 : 0 ;
	// the barcode salt lives above the 2k code bits of the 64-bit directory key (t4_index_key): 32 barcode bits need 2k <= 31
	if ( v && s && s->k > 15 )
	{
		set_err( "barcode-salted index needs k <= 15" ) ;
		return T4_E_UNSUPPORTED ;
	}
	return put_field( s, offsetof( T4Stream, considerBarcode ), &v, sizeof( int ) ) ;
}
int T4_API( seqset_set_is_long )( t4_seqset *s, int on )
{
	if ( on )
	{
		set_err( "isLongSeqSet (reads > 200 bp as the first read) is not supported" ) ;
		return T4_E_UNSUPPORTED ;
	}
	return check( s ) ;
}
int T4_API( seqset_size )( t4_seqset *s )
{
	T4Stream st ;
	int r = get_stream( s, &st ) ;
	if ( r ) return r ;
	return st.nSeqs ;
}
int T4_API( seqset_kmer_length )( t4_seqset *s )
{
	T4Stream st ;
	int r = get_stream( s, &st ) ;
	if ( r ) return r ;
	return st.kmerLength ;
}

// run one op on one stream through the staging buffer.  extra: bytes copied in after the op record;
// outBytes: bytes copied back from stage + outAt.
static int run_single( T4Op &op, const void *extra, size_t extraBytes, size_t outAt, void *outHost, size_t outBytes, size_t totalStage )
{
	int r = ensure_stage( totalStage ) ;
	if ( r ) return r ;
	// patch relative pointers: callers fill read/name/out as offsets from the stage start
	u64 b = (u64)(uintptr_t)E.stage ;
	if ( op.read ) op.read += b ;
	if ( op.name ) op.name += b ;
	if ( op.out ) op.out += b ;
	if ( op.out2 ) op.out2 += b ;
	r = h2d( E.stage, &op, sizeof( T4Op ) ) ;
	if ( r ) return r ;
	if ( extraBytes )
	{
		r = h2d( E.stage + sizeof( T4Op ), extra, extraBytes ) ;
		if ( r ) return r ;
	}
	r = launch_ops( T4K_STREAM, (T4Op *)E.stage, 1, 0 ) ;
	if ( r ) return r ;
	r = dsync() ;
	if ( r ) return r ;
	r = d2h( &op, E.stage, sizeof( T4Op ) ) ;
	if ( r ) return r ;
	if ( outBytes )
		r = d2h( outHost, E.stage + outAt, outBytes ) ;
	if ( op.ret < T4_E_BASE )
		set_err( "device-side error " + std::to_string( op.ret ) ) ;
	return r ;
}

static int read_ok( const char *read, int *len )
{
	size_t n = strlen( read ) ;
	if ( n > T4_DEV_MAX_READ )
	{
		set_err( "read longer than the device limit" ) ;
		return T4_E_UNSUPPORTED ;
	}
	*len = (int)n ;
	return 0 ;
}

int T4_API( seqset_add_read )( t4_seqset *s, const char *read, const char *gene_name, int *strand_inout, int barcode,
	int min_kmer_count, int repetitive, double sim_threshold )
{
	int r = check( s ) ;
	if ( r ) return r ;
	int len ;
	r = read_ok( read, &len ) ;
	if ( r ) return r ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = s->off ;
	op.op = T4_OP_ADD_READ ;
	op.read = sizeof( T4Op ) ;
	op.len = len ;
	op.strand = *strand_inout ;
	op.barcode = barcode ;
	op.minKmerCount = min_kmer_count ;
	op.repetitive = repetitive ;
	op.thr = sim_threshold ;
	strncpy( op.gene, gene_name ? gene_name : "", 7 ) ;
	r = run_single( op, read, len + 1, 0, 0, 0, sizeof( T4Op ) + len + 16 ) ;
	if ( r ) return r ;
	*strand_inout = op.strandOut ;
	return op.ret ;
}

int T4_API( seqset_repeat_add_read )( t4_seqset *s, const char *read )
{
	int r = check( s ) ;
	if ( r ) return r ;
	int len ;
	r = read_ok( read, &len ) ;
	if ( r ) return r ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = s->off ;
	op.op = T4_OP_REPEAT ;
	op.read = sizeof( T4Op ) ;
	op.len = len ;
	r = run_single( op, read, len + 1, 0, 0, 0, sizeof( T4Op ) + len + 16 ) ;
	if ( r ) return r ;
	return op.ret ;
}

int T4_API( seqset_input_novel_read )( t4_seqset *s, const char *id, const char *read, int strand, int barcode )
{
	int r = check( s ) ;
	if ( r ) return r ;
	int len ;
	r = read_ok( read, &len ) ;
	if ( r ) return r ;
	int nl = (int)strlen( id ) ;
	std::vector<char> extra( len + 1 + nl + 1 ) ;
	memcpy( extra.data(), read, len + 1 ) ;
	memcpy( extra.data() + len + 1, id, nl + 1 ) ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = s->off ;
	op.op = T4_OP_INPUT_NOVEL ;
	op.read = sizeof( T4Op ) ;
	op.name = sizeof( T4Op ) + len + 1 ;
	op.nameLen = nl ;
	op.len = len ;
	op.strand = strand ;
	op.barcode = barcode ;
	r = run_single( op, extra.data(), extra.size(), 0, 0, 0, sizeof( T4Op ) + extra.size() + 16 ) ;
	if ( r ) return r ;
	return op.ret ;
}

int T4_API( seqset_update_all_consensus )( t4_seqset *s )
{
	int r = check( s ) ;
	if ( r ) return r ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = s->off ;
	op.op = T4_OP_UPDATE_ALL ;
	r = run_single( op, 0, 0, 0, 0, 0, sizeof( T4Op ) ) ;
	if ( r ) return r ;
	return op.ret < T4_E_BASE ? op.ret : 0 ;
}

int T4_API( seqset_change_kmer_length )( t4_seqset *s, int kl )
{
	int r = check( s ) ;
	if ( r ) return r ;
	if ( kl < 2 || kl > 31 )
		return T4_E_INVAL ;
	if ( kl > 15 )
	{
		T4Stream st ;
		r = get_stream( s, &st ) ;
		if ( r ) return r ;
		if ( st.considerBarcode )
		{
			set_err( "barcode-salted index needs k <= 15" ) ;
			return T4_E_UNSUPPORTED ;
		}
	}
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = s->off ;
	op.op = T4_OP_CHANGE_K ;
	op.kl = kl ;
	r = run_single( op, 0, 0, 0, 0, 0, sizeof( T4Op ) ) ;
	if ( r ) return r ;
	s->k = kl ;
	return op.ret < T4_E_BASE ? op.ret : 0 ;
}

int T4_API( seqset_release_finished_barcode )( t4_seqset *s, int barcode, int contig_min_cov )
{
	int r = check( s ) ;
	if ( r ) return r ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = s->off ;
	op.op = T4_OP_RELEASE_BARCODE ;
	op.barcode = barcode ;
	op.minKmerCount = contig_min_cov ;
	r = run_single( op, 0, 0, 0, 0, 0, sizeof( T4Op ) ) ;
	if ( r ) return r ;
	return op.ret < T4_E_BASE ? op.ret : 0 ;
}

int T4_API( seqset_release_shallow_contigs )( t4_seqset *s, int min_cov )
{
	int r = check( s ) ;
	if ( r ) return r ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = s->off ;
	op.op = T4_OP_RELEASE_SHALLOW ;
	op.minKmerCount = min_cov ;
	r = run_single( op, 0, 0, 0, 0, 0, sizeof( T4Op ) ) ;
	if ( r ) return r ;
	return op.ret < T4_E_BASE ? op.ret : 0 ;
}

// SeqSet::InputNovelFa (SeqSet.hpp:2986): ReadFiles (kseq) semantics -- id = header up to the first white space,
// sequence lines concatenated.
int T4_API( seqset_input_novel_fa )( t4_seqset *s, const char *filename )
{
	int r = check( s ) ;
	if ( r ) return r ;
	FILE *fp = fopen( filename, "r" ) ;
	if ( !fp )
	{
		set_err( std::string( "cannot open " ) + filename ) ;
		return T4_E_INVAL ;
	}
	std::string id, seq, line ;
	int n = 0 ;
	bool have = false ;
	char buf[4096] ;
	auto flush = [&]() -> int
	{
		if ( !have )
			return 0 ;
		have = false ;
		int rr = T4_API( seqset_input_novel_read )( s, id.c_str(), seq.c_str(), 1, -1 ) ;
		if ( rr < T4_E_BASE )
			return rr ;
		++n ;
		return 0 ;
	} ;
	while ( fgets( buf, sizeof( buf ), fp ) )
	{
		line = buf ;
		while ( !line.empty() && ( line.back() == '\n' || line.back() == '\r' ) )
			line.pop_back() ;
		if ( !line.empty() && line[0] == '>' )
		{
			if ( ( r = flush() ) )
				break ;
			size_t e = line.find_first_of( " \t" ) ;
			id = line.substr( 1, e == std::string::npos ? std::string::npos : e - 1 ) ;
			seq.clear() ;
			have = true ;
		}
		else if ( have )
			seq += line ;
	}
	if ( !r )
		r = flush() ;
	fclose( fp ) ;
	return r ? r : n ;
}

int T4_API( seqset_contig_flags )( t4_seqset *s, int slot )
{
	T4Stream st ;
	int r = get_stream( s, &st ) ;
	if ( r ) return r ;
	if ( slot < 0 || slot >= st.nSeqs )
		return -1 ;
	T4Contig k ;
	r = d2h( &k, E.A + st.seqsOff + (size_t)slot * sizeof( T4Contig ), sizeof( k ) ) ;
	if ( r ) return r ;
	if ( !k.consOff )
		return -1 ;
	return ( k.flags & T4_CF_NOINDEX ) ? T4_CONTIG_PURGED : 0 ;
}

int T4_API( seqset_get_hits )( t4_seqset *s, const char *read, int strand, int barcode, int allow_total_skip, int32_t *hits, int cap )
{
	int r = check( s ) ;
	if ( r ) return r ;
	int len ;
	r = read_ok( read, &len ) ;
	if ( r ) return r ;
	size_t outAt = ( sizeof( T4Op ) + len + 1 + 63 ) & ~(size_t)63 ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = s->off ;
	op.op = T4_OP_GET_HITS ;
	op.read = sizeof( T4Op ) ;
	op.len = len ;
	op.strand = strand ;
	op.barcode = barcode ;
	op.repetitive = allow_total_skip ;
	op.out = outAt ;
	op.outCap = cap ;
	// two-step: the count first (cap may be too small), then the copy of min(count, cap)
	r = run_single( op, read, len + 1, 0, 0, 0, outAt + (size_t)cap * 20 + 64 ) ;
	if ( r ) return r ;
	if ( op.ret > 0 )
	{
		int n = op.ret < cap ? op.ret : cap ;
		r = d2h( hits, E.stage + outAt, (size_t)n * 20 ) ;
		if ( r ) return r ;
	}
	return op.ret ;
}

int T4_API( seqset_get_overlaps )( t4_seqset *s, const char *read, int strand, int barcode, int skip_repeats, int32_t *overlaps,
	double *similarity, int cap )
{
	int r = check( s ) ;
	if ( r ) return r ;
	int len ;
	r = read_ok( read, &len ) ;
	if ( r ) return r ;
	size_t outAt = ( sizeof( T4Op ) + len + 1 + 63 ) & ~(size_t)63 ;
	size_t out2At = outAt + (size_t)cap * 32 ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = s->off ;
	op.op = T4_OP_GET_OVERLAPS ;
	op.read = sizeof( T4Op ) ;
	op.len = len ;
	op.strand = strand ;
	op.barcode = barcode ;
	op.repetitive = skip_repeats ;
	op.out = outAt ;
	op.out2 = out2At ;
	op.outCap = cap ;
	r = run_single( op, read, len + 1, 0, 0, 0, out2At + (size_t)cap * 8 + 64 ) ;
	if ( r ) return r ;
	if ( op.ret > 0 )
	{
		int n = op.ret < cap ? op.ret : cap ;
		r = d2h( overlaps, E.stage + outAt, (size_t)n * 32 ) ;
		if ( r ) return r ;
		r = d2h( similarity, E.stage + out2At, (size_t)n * 8 ) ;
		if ( r ) return r ;
	}
	return op.ret ;
}

// ---- contigs back to the host -------------------------------------------------
struct HostContigs
{
	T4Stream st ;
	std::vector<T4Contig> ct ;
	std::vector<u64> off ;
	std::vector<char> data ;
} ;

static int fetch_contigs( t4_seqset *s, HostContigs &hc )
{
	int r = get_stream( s, &hc.st ) ;
	if ( r ) return r ;
	int n = hc.st.nSeqs ;
	hc.ct.resize( n ) ;
	hc.off.assign( n + 1, 0 ) ;
	if ( n == 0 )
		return 0 ;
	r = d2h( hc.ct.data(), E.A + hc.st.seqsOff, (size_t)n * sizeof( T4Contig ) ) ;
	if ( r ) return r ;
	u64 tot = 0 ;
	for ( int i = 0 ; i < n ; ++i )
	{
		hc.off[i] = tot ;
		if ( hc.ct[i].consOff )
			tot += ( 17ull * hc.ct[i].len + hc.ct[i].nameLen + 15 ) & ~15ull ;
	}
	hc.off[n] = tot ;
	hc.data.resize( tot ) ;
	if ( tot == 0 )
		return 0 ;
	DevBuf m ;
	T4Contig *dct ;
	u64 *doff ;
	char *dout ;
	m.add( dct, (size_t)n * sizeof( T4Contig ) ) ;
	m.add( doff, ( n + 1 ) * 8 ) ;
	m.add( dout, tot ) ;
	r = ensure_stage( m.bytes ) ;
	if ( r ) return r ;
	m.place( E.stage ) ;
	if ( ( r = h2d( dct, hc.ct.data(), (size_t)n * sizeof( T4Contig ) ) ) || ( r = h2d( doff, hc.off.data(), ( n + 1 ) * 8 ) )
		|| ( r = launch_blocks( T4_KERNEL( t4_gather_kernel, t4_gather_block ), n, 128, E.A, dct, doff, dout, n ) ) )
		return r ;
	return d2h( hc.data.data(), dout, tot ) ;
}

// SeqSet::Output (SeqSet.hpp:10939-10994)
static int output_to( t4_seqset *s, FILE *fp, const char *const *barcode_names, int n_barcode_names )
{
	HostContigs hc ;
	int r = fetch_contigs( s, hc ) ;
	if ( r ) return r ;
	int n = hc.st.nSeqs ;
	std::string line ;
	for ( int i = 0 ; i < n ; ++i )
	{
		const T4Contig &k = hc.ct[i] ;
		if ( !k.consOff )
			continue ;
		const char *o = hc.data.data() + hc.off[i] ;
		std::string cons( o, k.len ) ;
		std::string name( o + 17ull * k.len, k.nameLen ) ;
		const int32_t *pw = (const int32_t *)( o + k.len ) ;
		// posWeight columns start at byte k.len: may be unaligned in the packed buffer -> copy
		std::vector<int32_t> w( 4 * (size_t)k.len ) ;
		memcpy( w.data(), (const void *)pw, 16ull * k.len ) ;
		if ( barcode_names == NULL || k.barcode == -1 || k.barcode >= n_barcode_names )
			fprintf( fp, ">assemble%d %s\n%s\n", i, name.c_str(), cons.c_str() ) ;
		else
			fprintf( fp, ">%s_%d %s\n%s\n", barcode_names[k.barcode], i, name.c_str(), cons.c_str() ) ;
		for ( int c = 0 ; c < 4 ; ++c )
		{
			line.clear() ;
			char buf[16] ;
			for ( int j = 0 ; j < k.len ; ++j )
			{
				int m = snprintf( buf, sizeof( buf ), "%d ", w[4 * j + c] ) ;
				line.append( buf, m ) ;
			}
			line.push_back( '\n' ) ;
			fwrite( line.data(), 1, line.size(), fp ) ;
		}
	}
	return 0 ;
}

int T4_API( seqset_output )( t4_seqset *s, FILE *fp, const char *const *barcode_names, int n ) { return output_to( s, fp, barcode_names, n ) ; }

int T4_API( seqset_output_mem )( t4_seqset *s, char **buf, size_t *len )
{
	FILE *fp = open_memstream( buf, len ) ;
	if ( !fp )
		return T4_E_NOMEM ;
	int r = output_to( s, fp, NULL, 0 ) ;
	fclose( fp ) ;
	return r ;
}

void T4_API( free )( void *p ) { free( p ) ; }

int T4_API( seqset_get_contig )( t4_seqset *s, int slot, char *consensus, int consensus_cap, int32_t *pos_weight, char *name,
	int name_cap, int *barcode, int *num_read, int *min_left, int *min_right )
{
	T4Stream st ;
	int r = get_stream( s, &st ) ;
	if ( r ) return r ;
	if ( slot < 0 || slot >= st.nSeqs )
		return -1 ;
	T4Contig k ;
	r = d2h( &k, E.A + st.seqsOff + (size_t)slot * sizeof( T4Contig ), sizeof( k ) ) ;
	if ( r ) return r ;
	if ( !k.consOff )
		return -1 ;
	if ( consensus && consensus_cap > k.len )
	{
		r = d2h( consensus, E.A + k.consOff + k.lead, k.len ) ;
		if ( r ) return r ;
		consensus[k.len] = '\0' ;
	}
	if ( pos_weight )
	{
		r = d2h( pos_weight, E.A + k.pwOff + 16ull * k.lead, 16ull * k.len ) ;
		if ( r ) return r ;
	}
	if ( name && name_cap > 0 )
	{
		int m = k.nameLen < name_cap - 1 ? k.nameLen : name_cap - 1 ;
		r = d2h( name, E.A + k.nameOff, m ) ;
		if ( r ) return r ;
		name[m] = '\0' ;
	}
	if ( barcode ) *barcode = k.barcode ;
	if ( num_read ) *num_read = k.numRead ;
	if ( min_left ) *min_left = k.minLeftExtAnchor ;
	if ( min_right ) *min_right = k.minRightExtAnchor ;
	return k.len ;
}

// Order-independent checksum + count of all postings (test hook, mirrors oracle t4ref_index_checksum)
int64_t T4_API( seqset_index_checksum )( t4_seqset *s, uint64_t *checksum )
{
	T4Stream st ;
	int r = get_stream( s, &st ) ;
	if ( r ) return r ;
	std::vector<T4Dir> dir( st.dirCap ) ;
	r = d2h( dir.data(), E.A + st.dirOff, (size_t)st.dirCap * sizeof( T4Dir ) ) ;
	if ( r ) return r ;
	int64_t total = 0 ;
	uint64_t sum = 0 ;
	std::vector<u64> l ;
	u64 saltMask = ( st.kmerLength < 32 ) ? ( ( 1ull << ( 2 * st.kmerLength ) ) - 1 ) : ~0ull ;
	for ( u32 i = 0 ; i < st.dirCap ; ++i )
	{
		if ( dir[i].key == 0 || dir[i].cnt == 0 )
			continue ;
		l.resize( dir[i].cnt ) ;
		r = d2h( l.data(), E.A + dir[i].listOff, (size_t)dir[i].cnt * 8 ) ;
		if ( r ) return r ;
		u64 code = ( dir[i].key - 1 ) & saltMask ;
		for ( u32 j = 0 ; j < dir[i].cnt ; ++j )
		{
			uint64_t x = code * 0x9E3779B97F4A7C15ull ^ l[j] ;
			x ^= x >> 31 ; x *= 0xBF58476D1CE4E5B9ull ; x ^= x >> 29 ;
			sum += x ;
		}
		total += dir[i].cnt ;
	}
	*checksum = sum ;
	return total ;
}

// Every live column's equality byte against its posWeight counts (test hook of the t4_eq cache)
int64_t T4_API( test_check_eq_bytes )( t4_seqset *s, int64_t *bad )
{
	T4Stream st ;
	int r = get_stream( s, &st ) ;
	if ( r ) return r ;
	std::vector<T4Contig> ct( st.nSeqs ) ;
	if ( st.nSeqs && ( r = d2h( ct.data(), E.A + st.seqsOff, (size_t)st.nSeqs * sizeof( T4Contig ) ) ) )
		return r ;
	int64_t cols = 0, nbad = 0 ;
	std::vector<int32_t> pw ;
	std::vector<unsigned char> eq ;
	for ( const T4Contig &k : ct )
	{
		if ( !k.consOff )
			continue ;
		pw.resize( 4 * (size_t)k.len ) ;
		eq.resize( k.len ) ;
		if ( ( r = d2h( pw.data(), E.A + k.pwOff + 16ull * k.lead, 16ull * k.len ) )
			|| ( r = d2h( eq.data(), E.A + k.pwOff + 16ull * k.cap + k.lead, k.len ) ) )
			return r ;
		for ( int i = 0 ; i < k.len ; ++i )
			nbad += eq[i] != t4_eq_nibble( pw.data() + 4 * i ) ;
		cols += k.len ;
	}
	*bad = nbad ;
	return cols ;
}

// ---- host utilities -----------------------------------------------------------
// SeqSet::DnaToAa (SeqSet.hpp:638): standard code, '-' for codons with N
static char dna_to_aa( char a, char b, char c )
{
	if ( a == 'N' || b == 'N' || c == 'N' )
		return '-' ;
	static const char *tab = "KNKNTTTTRSRSIIMIQHQHPPPPRRRRLLLLEDEDAAAAGGGGVVVV_Y_YSSSS_CWCLFLF" ;
	return tab[16 * t4_nuc( a ) + 4 * t4_nuc( b ) + t4_nuc( c )] ;
}

// SeqSet::HasMotif (SeqSet.hpp:5029): note that the reference translates `read` itself for either strand
int T4_API( has_motif )( const char *read, int strand )
{
	if ( strand == 0 )
		return 0 ;
	int len = (int)strlen( read ) ;
	std::vector<char> aa( len + 1 ) ;
	int ret = 0 ;
	for ( int k = 0 ; k <= 2 ; ++k )
	{
		int i, j ;
		for ( i = k, j = 0 ; i + 2 < len ; i += 3, ++j )
			aa[j] = dna_to_aa( read[i], read[i + 1], read[i + 2] ) ;
		for ( i = 0 ; i + 2 < j ; ++i )
			if ( aa[i] == 'Y' && aa[i + 1] == 'Y' && aa[i + 2] == 'C' )
			{
				ret |= 2 ;
				break ;
			}
		for ( i = 0 ; i + 3 < j ; ++i )
			if ( ( aa[i] == 'F' || aa[i] == 'W' ) && aa[i + 1] == 'G' && aa[i + 3] == 'G' )
			{
				ret |= 1 ;
				break ;
			}
	}
	return ret ;
}

// SeqSet::ReverseComplementInPlace (SeqSet.hpp:2629)
void T4_API( reverse_complement_in_place )( char *seq, int len )
{
	int i, j ;
	for ( i = 0, j = len - 1 ; i < j ; ++i, --j )
	{
		char tmp = seq[j] ;
		seq[j] = ( seq[i] != 'N' ) ? t4_numToNuc( 3 - t4_nuc( seq[i] ) ) : 'N' ;
		seq[i] = ( tmp != 'N' ) ? t4_numToNuc( 3 - t4_nuc( tmp ) ) : 'N' ;
	}
	if ( i == j )
		seq[i] = ( seq[i] != 'N' ) ? t4_numToNuc( 3 - t4_nuc( seq[i] ) ) : 'N' ;
}

// ---- DP batch -------------------------------------------------------------------
int T4_API( dp_pos_weight_batch )( int n, const int32_t *t_weights, const int64_t *t_off, const char *p, const int64_t *p_off,
	int8_t *align_out, const int64_t *align_off, int32_t *score_out )
{
	int r = ensure_up() ;
	if ( r ) return r ;
	if ( n <= 0 )
		return 0 ;
	std::vector<i64> so( n + 1 ) ;
	i64 tot = 0 ;
	i64 alignTot = 0 ;
	for ( int i = 0 ; i < n ; ++i )
	{
		i64 lent = t_off[i + 1] - t_off[i], lenp = p_off[i + 1] - p_off[i] ;
		i64 d = lent > lenp ? lent - lenp : lenp - lent ;
		i64 W = 2 * T4_DP_BAND + 3 + d ;
		so[i] = tot ;
		tot += ( 8 * W + ( lenp + 1 ) * W + 15 ) & ~15ll ;
		i64 e = align_off[i] + lent + lenp + 2 ;
		if ( e > alignTot )
			alignTot = e ;
	}
	so[n] = tot ;
	size_t szT = (size_t)t_off[n] * 16, szP = (size_t)p_off[n], szO = ( n + 1 ) * 8 ;
	T4DpParams P ;
	P.n = n ;
	DevBuf m ;
	int *dT ;
	char *dP ;
	i64 *dTo, *dPo, *dAo, *dSo ;
	m.add( dT, szT + 16 ) ; m.add( dP, szP + 16 ) ; m.add( dTo, szO ) ; m.add( dPo, szO ) ; m.add( P.align, (size_t)alignTot + 16 ) ;
	m.add( dAo, szO ) ; m.add( P.score, (size_t)n * 4 ) ; m.add( P.scratch, (size_t)tot + 16 ) ; m.add( dSo, szO ) ;
	if ( ( r = m.alloc() ) )
		return r ;
	P.tw = dT ; P.p = dP ; P.tOff = dTo ; P.pOff = dPo ; P.alignOff = dAo ; P.scratchOff = dSo ;
	if ( ( r = h2d( dT, t_weights, szT ) ) || ( r = h2d( dP, p, szP ) ) || ( r = h2d( dTo, t_off, szO ) ) || ( r = h2d( dPo, p_off, szO ) )
		|| ( r = h2d( dAo, align_off, szO ) ) || ( r = h2d( dSo, so.data(), szO ) )
		|| ( r = launch_items( T4_KERNEL( t4_dp_kernel, t4_dp_one ), P, n, 64 ) ) || ( r = dsync() ) )
		return r ;
	if ( ( r = d2h( align_out, P.align, alignTot ) ) || ( r = d2h( score_out, P.score, (size_t)n * 4 ) ) )
		return r ;
	return 0 ;
}

// The hot-path DP routines on n equal-length problems (problem i: columns / bases off[i]..off[i+1)).
// variant 0: t4_dp_equal; variant 1: w_dp_equal_half; variant 2: w_side_pair (1 and 2: product build only).
int T4_API( dp_hot_path_batch )( int n, int variant, const int32_t *t_weights, const int64_t *off, const char *p, int8_t *align_out,
	const int64_t *align_off, int32_t *score_out )
{
	int r = ensure_up() ;
	if ( r ) return r ;
	if ( n <= 0 )
		return 0 ;
	if ( variant < 0 || variant > 2 )
		return T4_E_INVAL ;
#if !T4_CUDA
	if ( variant != 0 )
	{
		set_err( "the warp DP routines exist only in the CUDA build" ) ;
		return T4_E_UNSUPPORTED ;
	}
#endif
	std::vector<i64> so( n + 1 ) ;
	i64 tot = 0, alignTot = 0 ;
	for ( int i = 0 ; i < n ; ++i )
	{
		i64 len = off[i + 1] - off[i] ;
		so[i] = tot ;
		i64 stride = len / 16 + 2 ;
		tot += 26 * stride + ( 2 * ( 2 * len + 8 ) + 3 ) / 4 + len + 8 ; // u32 words: traceback of both halves, edit strings, act32 of variant 0
		if ( variant == 2 && ( align_off[i] & 3 ) )
			return T4_E_INVAL ;
		i64 e = align_off[i] + ( ( variant == 2 && 2 * len + 2 < 16 ) ? 16 : 2 * len + 2 ) ;
		if ( e > alignTot )
			alignTot = e ;
	}
	so[n] = tot ;
	size_t szT = (size_t)off[n] * 16, szP = (size_t)off[n], szO = (size_t)( n + 1 ) * 8 ;
	DevBuf m ;
	int *dT, *dS ;
	char *dP ;
	i64 *dOff, *dAo, *dSo ;
	signed char *dA ;
	u32 *dScr ;
	m.add( dT, szT + 16 ) ; m.add( dP, szP + 16 ) ; m.add( dOff, szO ) ; m.add( dA, (size_t)alignTot + 16 ) ; m.add( dAo, szO ) ;
	m.add( dS, (size_t)n * 4 ) ; m.add( dScr, (size_t)tot * 4 + 16 ) ; m.add( dSo, szO ) ;
	if ( ( r = m.alloc() ) || ( r = h2d( dT, t_weights, szT ) ) || ( r = h2d( dP, p, szP ) ) || ( r = h2d( dOff, off, szO ) )
		|| ( r = h2d( dAo, align_off, szO ) ) || ( r = h2d( dSo, so.data(), szO ) ) )
		return r ;
#if T4_CUDA
	t4_dp_hot_kernel<<<variant == 2 ? ( n + 1 ) / 2 : n, 32>>>( n, variant, dT, dOff, dP, dA, dAo, dS, dScr, dSo ) ;
	CK( cudaGetLastError() ) ;
	CK( cudaDeviceSynchronize() ) ;
#else
	for ( int i = 0 ; i < n ; ++i )
		dS[i] = t4_dp_equal( dT + 4 * off[i], dP + off[i], (int)( off[i + 1] - off[i] ), dA + align_off[i], dScr + so[i], false, 0 ) ;
#endif
	if ( ( r = d2h( align_out, dA, alignTot ) ) || ( r = d2h( score_out, dS, (size_t)n * 4 ) ) )
		return r ;
	return 0 ;
}

// ---- workloads / batch -------------------------------------------------------------
static t4_workload *workload_upload_impl( const t4_read_desc *descs, int64_t n, const char *read_pool, size_t pool_bytes,
	const char *const *names, int n_names, bool persistent )
{
	if ( ensure_up() )
		return 0 ;
	std::vector<u32> noff( n_names + 1 ) ;
	std::string npool ;
	for ( int i = 0 ; i < n_names ; ++i )
	{
		noff[i] = (u32)npool.size() ;
		npool += names[i] ;
	}
	noff[n_names] = (u32)npool.size() ;
	// 2-bit packed copy of the reads, fixed stride (the longest supported read of the workload)
	int maxLen = 0 ;
	{
		// one pass over the record array (64 B stride); a few host threads, this sits inside the e2e path
		const int nth = n > ( 1 << 18 ) ? 8 : 1 ;
		std::vector<int> part( nth, 0 ) ;
		std::vector<std::thread> th ;
		for ( int t = 0 ; t < nth ; ++t )
			th.emplace_back( [&, t]() {
				int m = 0 ;
				for ( int64_t i = n * t / nth ; i < n * ( t + 1 ) / nth ; ++i )
					if ( descs[i].len > m && descs[i].len <= T4_DEV_MAX_READ )
						m = descs[i].len ;
				part[t] = m ;
			} ) ;
		for ( auto &x : th )
			x.join() ;
		for ( int t = 0 ; t < nth ; ++t )
			if ( part[t] > maxLen )
				maxLen = part[t] ;
	}
	const u64 packStride = t4_pack_words( maxLen ) ;
	t4_workload *w = new t4_workload ;
	memset( w, 0, sizeof( *w ) ) ;
	w->persistent = persistent ;
	w->nDescs = n ;
	w->poolBytes = pool_bytes ;
	w->nNames = n_names ;
	w->packStride = packStride ;
	DevBuf m ;
	u32 *dNoff, *dOdd ;
	char *dNpool ;
	m.add( w->descs, (size_t)n * sizeof( t4_read_desc ) ) ; m.add( w->pool, pool_bytes + 16 ) ; m.add( w->names, sizeof( T4Names ) ) ;
	m.add( dNoff, ( n_names + 1 ) * 4 ) ; m.add( dNpool, npool.size() + 16 ) ; m.add( w->ret, (size_t)n * 4 ) ; m.add( w->strands, (size_t)n ) ;
	m.add( w->rescue, (size_t)n * 4 ) ; m.add( w->rescueList, (size_t)n * 4 ) ; m.add( w->good, (size_t)n ) ; m.add( w->info, (size_t)n * 4 ) ;
	m.add( w->events, (size_t)n ) ; m.add( w->packed, (size_t)n * packStride * 8 + 16 ) ; m.add( dOdd, 256 ) ;
	if ( persistent )
	{
		if ( E.wlCap < m.bytes )
		{
			if ( E.wl )
				dfree( E.wl ) ;
			E.wl = 0 ;
			E.wlCap = 0 ;
			void *p = 0 ;
			size_t c = m.bytes + m.bytes / 4 ;
			if ( dmalloc( &p, c ) )
			{
				delete w ;
				return 0 ;
			}
			E.wl = (char *)p ;
			E.wlCap = c ;
		}
		m.place( E.wl ) ;
	}
	else if ( m.alloc() )
	{
		delete w ;
		return 0 ;
	}
	T4Names hn ;
	hn.pool = (u64)(uintptr_t)dNpool ;
	hn.off = (u64)(uintptr_t)dNoff ;
	hn.n = n_names ;
	hn.pad = 0 ;
	bool ok = !h2d( w->descs, descs, (size_t)n * sizeof( t4_read_desc ) ) && !h2d( w->pool, read_pool, pool_bytes ) && !h2d( w->names, &hn, sizeof( hn ) )
		&& !h2d( dNoff, noff.data(), ( n_names + 1 ) * 4 ) && !h2d( dNpool, npool.data(), npool.size() ) ;
	// pack on the device (the host API takes ASCII reads like the reference; they cross PCIe once, as ASCII)
	u32 odd = 0 ;
	if ( ok && n > 0 && packStride > 0 )
	{
		T4PackReadsParams P ;
		P.descs = w->descs ; P.n = n ; P.pool = w->pool ; P.packStride = packStride ; P.wMax = (int)t4_pack_w( maxLen ) ;
		P.packed = w->packed ; P.odd = dOdd ;
		ok = !dzero( dOdd, 4 ) && !launch_items( T4_KERNEL( t4_pack_reads_kernel, t4_pack_read_word ), P, n * P.wMax, 256 ) && !d2h( &odd, dOdd, 4 ) ;
		if ( !ok )
			set_err( "packing the reads failed" ) ;
	}
	if ( !ok )
	{
		delete w ;
		return 0 ;
	}
	w->buf = m.keep() ;
	w->bytes = m.bytes ;
	w->usePacked = ( odd == 0 && n > 0 && packStride > 0 ) ;
	return w ;
}

t4_workload *T4_API( workload_upload )( const t4_read_desc *descs, int64_t n, const char *read_pool, size_t pool_bytes,
	const char *const *names, int n_names )
{
	return workload_upload_impl( descs, n, read_pool, pool_bytes, names, n_names, false ) ;
}

void T4_API( workload_free )( t4_workload *w )
{
	if ( !w )
		return ;
	if ( w->ops )
		dfree( w->ops ) ;
	if ( !w->persistent )
		dfree( w->buf ) ;
	delete w ;
}

static int build_ops( t4_seqset *const *sets, int n_sets, const t4_run_cfg *cfg, t4_workload *w, const int64_t *desc_off, int opcode,
	std::vector<T4Op> &ops )
{
	ops.resize( n_sets ) ;
	for ( int j = 0 ; j < n_sets ; ++j )
	{
		int r = check( sets[j] ) ;
		if ( r ) return r ;
		// launch order = reverse stream order: the hardware hands out CTAs in block order, and in a sorted read list the
		// late shards (low-abundance, diverse reads) are the expensive ones (measured 1-20 ms for the first third of the
		// shards vs 150-700 ms for the last third) -- longest-first keeps the tail of the launch short
		T4Op &op = ops[n_sets - 1 - j] ;
		memset( &op, 0, sizeof( op ) ) ;
		i64 lo = desc_off[j], hi = desc_off[j + 1] ;
		if ( lo < 0 || hi < lo || hi > w->nDescs )
		{
			set_err( "desc_off out of range" ) ;
			return T4_E_INVAL ;
		}
		op.streamOff = sets[j]->off ;
		op.op = opcode ;
		op.n = (int)( hi - lo ) ;
		op.desc = (u64)(uintptr_t)( w->descs + lo ) ;
		op.pool = (u64)(uintptr_t)w->pool ;
		op.names = (u64)(uintptr_t)w->names ;
		op.retCodes = (u64)(uintptr_t)( w->ret + lo ) ;
		op.strands = (u64)(uintptr_t)( w->strands + lo ) ;
		op.rescueRet = (u64)(uintptr_t)( w->rescue + lo ) ;
		op.rescueList = (u64)(uintptr_t)( w->rescueList + lo ) ;
		op.good = (u64)(uintptr_t)( w->good + lo ) ;
		op.info = (u64)(uintptr_t)( w->info + lo ) ;
		op.events = (u64)(uintptr_t)( w->events + lo ) ;
		if ( w->usePacked )
		{
			op.packed = (u64)(uintptr_t)( w->packed + (u64)lo * w->packStride ) ;
			op.packStride = w->packStride ;
		}
		if ( cfg )
			op.cfg = *cfg ;
	}
	return 0 ;
}

static int ensure_ops( t4_workload *w, int n )
{
	if ( n <= w->opCap )
		return 0 ;
	if ( w->ops )
		dfree( w->ops ) ;
	void *p = 0 ;
	int r = dmalloc( &p, (size_t)n * sizeof( T4Op ) ) ;
	if ( r ) return r ;
	w->ops = (T4Op *)p ;
	w->opCap = n ;
	return 0 ;
}

int T4_API( streams_run_resident )( t4_seqset *const *sets, int n_sets, const t4_run_cfg *cfg, t4_workload *w, const int64_t *desc_off,
	void *cuda_stream )
{
	if ( !w || n_sets <= 0 )
		return T4_E_INVAL ;
	std::vector<T4Op> ops ;
	int r = build_ops( sets, n_sets, cfg, w, desc_off, T4_OP_RUN_LOOP, ops ) ;
	if ( r ) return r ;
	r = ensure_ops( w, n_sets ) ;
	if ( r ) return r ;
	w->ran = true ;
	r = h2d_async( w->ops, ops.data(), (size_t)n_sets * sizeof( T4Op ), cuda_stream ) ;
	if ( r ) return r ;
	return launch_ops( T4K_STREAM, w->ops, n_sets, cuda_stream ) ;
}

// ---- batch probe over frozen sets (t4_probe.cuh) ---------------------------------------------------
struct t4_hits
{
	i64 maxReads ;
	size_t keyCap ;
	char *buf ;            // one device allocation
	u64 *keys, *hitOff, *ord, *ctrl ;
	u32 *hitCnt, *hitFlags ;
	u64 *dStreamOff ;      // grow-only side buffers: stream offsets and desc_off of the last call
	i64 *dDescOff ;
	int setCap ;
	i64 nReads ;           // of the last probe
	int kLast ;
} ;

t4_hits *T4_API( hits_create )( int64_t max_reads, size_t max_hits )
{
	if ( ensure_up() || max_reads <= 0 )
		return 0 ;
	t4_hits *h = new t4_hits ;
	memset( h, 0, sizeof( *h ) ) ;
	h->maxReads = max_reads ;
	h->keyCap = max_hits ;
	DevBuf m ;
	m.add( h->keys, max_hits * 8 + 16 ) ; m.add( h->hitOff, (size_t)max_reads * 8 ) ; m.add( h->ord, (size_t)max_reads * 8 ) ;
	m.add( h->hitCnt, (size_t)max_reads * 4 ) ; m.add( h->hitFlags, (size_t)max_reads * 4 ) ; m.add( h->ctrl, 256 ) ;
	if ( m.alloc() || dzero( h->ctrl, 64 ) )
	{
		delete h ;
		return 0 ;
	}
	h->buf = m.keep() ;
	return h ;
}

void T4_API( hits_free )( t4_hits *h )
{
	if ( !h )
		return ;
	dfree( h->buf ) ;
	if ( h->dStreamOff ) dfree( h->dStreamOff ) ;
	if ( h->dDescOff ) dfree( h->dDescOff ) ;
	delete h ;
}

int T4_API( streams_get_hits )( t4_seqset *const *sets, int n_sets, t4_workload *w, const int64_t *desc_off, int allow_total_skip,
	void *cuda_stream, t4_hits *h )
{
	if ( !w || !h || n_sets <= 0 )
		return T4_E_INVAL ;
	const i64 n = desc_off[n_sets] - desc_off[0] ;
	if ( desc_off[0] != 0 || n > w->nDescs || n > h->maxReads )
	{
		set_err( "t4_streams_get_hits: desc_off must start at 0 and fit the workload and the hit buffer" ) ;
		return T4_E_INVAL ;
	}
	std::vector<u64> so( n_sets ) ;
	for ( int j = 0 ; j < n_sets ; ++j )
	{
		int r = check( sets[j] ) ;
		if ( r ) return r ;
		so[j] = sets[j]->off ;
	}
	if ( n_sets > h->setCap )
	{
		if ( h->dStreamOff ) dfree( h->dStreamOff ) ;
		if ( h->dDescOff ) dfree( h->dDescOff ) ;
		h->dStreamOff = 0 ; h->dDescOff = 0 ; h->setCap = 0 ;
		void *a = 0, *b = 0 ;
		int r = dmalloc( &a, (size_t)n_sets * 8 ) ;
		if ( !r ) r = dmalloc( &b, (size_t)( n_sets + 1 ) * 8 ) ;
		if ( r )
		{
			if ( a ) dfree( a ) ;
			return r ;
		}
		h->dStreamOff = (u64 *)a ; h->dDescOff = (i64 *)b ; h->setCap = n_sets ;
	}
	h->nReads = n ;
#if T4_CUDA
	cudaStream_t cs = (cudaStream_t)cuda_stream ;
	CK( cudaMemcpyAsync( h->dStreamOff, so.data(), (size_t)n_sets * 8, cudaMemcpyHostToDevice, cs ) ) ;
	CK( cudaMemcpyAsync( h->dDescOff, desc_off, (size_t)( n_sets + 1 ) * 8, cudaMemcpyHostToDevice, cs ) ) ;
	CK( cudaMemsetAsync( h->ctrl, 0, 64, cs ) ) ;
	if ( n == 0 )
		return 0 ;
	t4_bucket_kernel<<<n_sets, 128, 0, cs>>>( w->descs, h->dDescOff, h->ord ) ;
	CK( cudaGetLastError() ) ;
	T4ProbeParams P ;
	P.A = E.A ;
	P.streamOff = h->dStreamOff ;
	P.descs = w->descs ;
	P.packed = w->packed ;
	P.packStride = w->packStride ;
	P.ord = h->ord ;
	P.nReads = n ;
	P.keys = h->keys ;
	P.keyCap = h->keyCap ;
	P.hitOff = h->hitOff ;
	P.hitCnt = h->hitCnt ;
	P.hitFlags = h->hitFlags ;
	P.ctrl = h->ctrl ;
	P.allowTotalSkip = allow_total_skip ? 1 : 0 ;
	// registers bounded for 24 resident warps per SM, 2 directory probes in flight per lane
	void ( *const probeKernel )( T4ProbeParams ) = t4_probe_kernel<24, 2> ;
	static int probeBlocks = 0 ;
	const size_t probeSmem = sizeof( T4ProbeWarp ) * T4P_WARPS ;
	if ( probeBlocks == 0 )
	{
		int perSm = 0 ;
		CK( cudaFuncSetAttribute( probeKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)probeSmem ) ) ;
		CK( cudaOccupancyMaxActiveBlocksPerMultiprocessor( &perSm, probeKernel, 32 * T4P_WARPS, probeSmem ) ) ;
		probeBlocks = ( perSm > 0 ? perSm : 1 ) * E.sms ; // persistent: one wave, a multiple of the SM count
	}
	i64 need = ( n + T4P_WARPS - 1 ) / T4P_WARPS ;
	int blocks = need < probeBlocks ? (int)need : probeBlocks ;
	probeKernel<<<blocks, 32 * T4P_WARPS, probeSmem, cs>>>( P ) ;
	CK( cudaGetLastError() ) ;
#else
	// TEST EMULATION: the same result through the stream engine's own GetHitsFromRead, one read at a time
	(void)cuda_stream ;
	memcpy( h->dStreamOff, so.data(), (size_t)n_sets * 8 ) ;
	memset( h->ctrl, 0, 64 ) ;
	T4Smem *sm = new T4Smem ;
	u64 top = 0 ;
	for ( int j = 0 ; j < n_sets ; ++j )
		for ( i64 i = desc_off[j] ; i < desc_off[j + 1] ; ++i )
		{
			T4Ctx cx = t4_ctx( E.A, so[j], sm, 0, 1 ) ;
			const t4_read_desc &d = w->descs[i] ;
			h->hitOff[i] = top ;
			h->hitCnt[i] = 0 ;
			h->hitFlags[i] = 0 ;
			if ( d.len > T4_DEV_MAX_READ )
				++h->ctrl[7] ;
			if ( d.len > T4_DEV_MAX_READ || d.len < cx.st->kmerLength )
				continue ;
			for ( int x = 0 ; x < T4_N_COUNTERS ; ++x )
				sm->ctr[x] = 0 ;
			c_load_read_packed( cx, w->packed + (u64)i * w->packStride, d.len ) ;
			int anyBig = 0 ;
			u32 H = c_get_hits( cx, d.len, d.strand_in, d.barcode, allow_total_skip != 0, &anyBig ) ;
			if ( top + H > h->keyCap )
			{
				h->ctrl[2] = 1 ;
				top += H ;
				continue ;
			}
			memcpy( h->keys + top, E.A + cx.st->keysAOff, (size_t)H * 8 ) ;
			h->hitCnt[i] = H ;
			h->hitFlags[i] = anyBig ? 1u : 0u ;
			top += H ;
			h->ctrl[3] += sm->ctr[2] ; h->ctrl[4] += sm->ctr[3] ; h->ctrl[5] += sm->ctr[4] ; h->ctrl[6] += sm->ctr[5] ;
		}
	h->ctrl[1] = top ;
	delete sm ;
#endif
	return 0 ;
}

// stats[0] hits emitted (sum c_j', keys written), [1] lookups executed, [2] postings read (sum c_j), [3] packed read bytes ceil(L/4),
// [4] algorithmic bytes by SURVEY.md 8d with the 8-byte key this kernel really writes: [3] + 8 [1] + 8 [2] + 8 [0],
// [5] the same with the survey's nominal 16-byte hit, [6] reads longer than T4_MAX_READ_LEN (skipped), [7] reads probed.
int T4_API( hits_stats )( t4_hits *h, uint64_t *stats )
{
	if ( !h )
		return T4_E_INVAL ;
	int r = dsync() ;
	if ( r ) return r ;
	u64 c[8] ;
	r = d2h( c, h->ctrl, 64 ) ;
	if ( r ) return r ;
	stats[0] = c[5] ; stats[1] = c[3] ; stats[2] = c[4] ; stats[3] = c[6] ;
	stats[4] = c[6] + 8 * c[3] + 8 * c[4] + 8 * c[5] ;
	stats[5] = c[6] + 8 * c[3] + 8 * c[4] + 16 * c[5] ;
	stats[6] = c[7] ;
	stats[7] = (u64)h->nReads ;
	if ( c[2] )
	{
		set_err( "hit buffer too small: " + std::to_string( c[1] ) + " keys needed" ) ;
		return T4_E_NOMEM ;
	}
	return 0 ;
}

// Hits of record i as int32[4] = { seqIdx, seqOffset, readOffset, strand }; hits removed by the barcode filter
// (SeqSet.hpp:1418) are dropped.  Order: by read position (forward pass first), postings order inside a k-mer.
int T4_API( hits_fetch )( t4_hits *h, int64_t record, int32_t *hits, int cap, int *flags )
{
	if ( !h || record < 0 || record >= h->nReads )
		return T4_E_INVAL ;
	int r = dsync() ;
	if ( r ) return r ;
	u64 off ;
	u32 cnt, fl ;
	if ( ( r = d2h( &off, h->hitOff + record, 8 ) ) || ( r = d2h( &cnt, h->hitCnt + record, 4 ) ) || ( r = d2h( &fl, h->hitFlags + record, 4 ) ) )
		return r ;
	if ( flags )
		*flags = (int)fl ;
	std::vector<u64> k( cnt ) ;
	if ( cnt && ( r = d2h( k.data(), h->keys + off, (size_t)cnt * 8 ) ) )
		return r ;
	int n = 0 ;
	for ( u32 i = 0 ; i < cnt ; ++i )
	{
		if ( k[i] == T4_KEY_INVALID )
			continue ;
		if ( n < cap )
		{
			hits[4 * n] = t4_key_idx( k[i] ) ;
			hits[4 * n + 1] = t4_key_b( k[i] ) ;
			hits[4 * n + 2] = t4_key_a( k[i] ) ;
			hits[4 * n + 3] = t4_key_strand( k[i] ) ;
		}
		++n ;
	}
	return n ;
}

// raw access for device-side consumers and tests: device pointers of the last probe
int T4_API( hits_device_buffers )( t4_hits *h, void **keys, void **hit_off, void **hit_cnt )
{
	if ( !h )
		return T4_E_INVAL ;
	if ( keys ) *keys = h->keys ;
	if ( hit_off ) *hit_off = h->hitOff ;
	if ( hit_cnt ) *hit_cnt = h->hitCnt ;
	return 0 ;
}

int T4_API( streams_error )( t4_seqset *const *sets, int n_sets ) ;

// ---- AssignRead pass over frozen sets (t4_assign.h; SURVEY.md 8f-2) ------------------------------------------------
struct t4_assign
{
	char *buf ;            // one device allocation: parameter block, op records, result arrays
	i64 nDescs ;
	int nSets ;
	T4AssignParams *dP ;
	int32_t *dAssign ;
	double *dSim ;
	u64 *dCursor ;
	std::vector<t4_seqset *> ext ;     // the extended sets (extendedSeq of main.cpp:2047), one per stage-1 set
	std::vector<t4_seqset *> workers ; // scratch-only streams of the ASSIGN launch
	uint32_t gen ;
} ;

void T4_API( assign_free )( t4_assign *a )
{
	if ( !a )
		return ;
	if ( a->buf ) dfree( a->buf ) ;
	for ( size_t i = 0 ; i < a->ext.size() ; ++i ) delete a->ext[i] ;
	for ( size_t i = 0 ; i < a->workers.size() ; ++i ) delete a->workers[i] ;
	delete a ;
}

t4_assign *T4_API( streams_assign_reads )( t4_seqset *const *sets, int n_sets, t4_workload *w, const int64_t *desc_off, int kmer_length,
	int n_workers, void *cuda_stream )
{
	if ( !w || !sets || !desc_off || n_sets <= 0 )
	{
		set_err( "t4_streams_assign_reads: bad argument" ) ;
		return 0 ;
	}
	const i64 n = desc_off[n_sets] ;
	if ( desc_off[0] != 0 || n > w->nDescs || n >= ( 1ll << 31 ) )
	{
		set_err( "t4_streams_assign_reads: desc_off must start at 0 and fit the workload" ) ;
		return 0 ;
	}
	if ( !w->ran )
	{
		set_err( "t4_streams_assign_reads: the workload holds no assembly results yet (t4_streams_run_resident comes first)" ) ;
		return 0 ;
	}
	for ( int j = 0 ; j < n_sets ; ++j )
		if ( check( sets[j] ) || desc_off[j + 1] < desc_off[j] )
		{
			set_err( "t4_streams_assign_reads: stale handle or unordered desc_off" ) ;
			return 0 ;
		}
	if ( n_workers <= 0 )
		n_workers = resident_workers() ;
	t4_assign *a = new t4_assign ;
	a->buf = 0 ; a->nDescs = n ; a->nSets = n_sets ; a->gen = g_gen ;
	a->ext.assign( n_sets, (t4_seqset *)0 ) ;
	a->workers.assign( n_workers, (t4_seqset *)0 ) ;
	// fresh sets with the constructor's defaults (SeqSet.hpp:2558-2576): the extended sets at the pass's k, the workers' shells
	if ( seqsets_create_impl( n_sets, kmer_length, 31, 0, a->ext.data() ) || seqsets_create_impl( n_workers, kmer_length, 31, 0, a->workers.data() ) )
	{
		T4_API( assign_free )( a ) ;
		return 0 ;
	}
	const size_t nn = (size_t)( n > 0 ? n : 1 ) ;
	DevBuf m ;
	T4Op *dOpsA, *dOpsB, *dOpsC ;
	u64 *dExt, *dSrc ;
	i64 *dDoff ;
	int32_t *dCnt, *dList, *dLead, *dSet ;
	m.add( a->dP, sizeof( T4AssignParams ) ) ; m.add( a->dCursor, 256 ) ; m.add( dOpsA, (size_t)n_sets * sizeof( T4Op ) ) ;
	m.add( dOpsB, (size_t)n_workers * sizeof( T4Op ) ) ; m.add( dOpsC, (size_t)n_sets * sizeof( T4Op ) ) ; m.add( dExt, (size_t)n_sets * 8 ) ;
	m.add( dSrc, (size_t)n_sets * 8 ) ; m.add( dDoff, (size_t)( n_sets + 1 ) * 8 ) ; m.add( dCnt, (size_t)n_sets * 4 ) ; m.add( dList, nn * 4 ) ;
	m.add( dLead, nn * 4 ) ; m.add( dSet, nn * 4 ) ; m.add( a->dAssign, nn * 32 ) ; m.add( a->dSim, nn * 8 ) ;
	if ( m.alloc() )
	{
		T4_API( assign_free )( a ) ;
		return 0 ;
	}
	T4AssignParams P ;
	memset( &P, 0, sizeof( P ) ) ;
	auto dp = []( const void *q ) { return (u64)(uintptr_t)q ; } ;
	P.descs = dp( w->descs ) ; P.pool = dp( w->pool ) ; P.ret = dp( w->ret ) ; P.strands = dp( w->strands ) ; P.rescue = dp( w->rescue ) ;
	P.list = dp( dList ) ; P.leader = dp( dLead ) ; P.slotSet = dp( dSet ) ; P.assign = dp( a->dAssign ) ; P.sim = dp( a->dSim ) ;
	P.extOff = dp( dExt ) ; P.srcOff = dp( dSrc ) ; P.descOff = dp( dDoff ) ; P.listCnt = dp( dCnt ) ; P.cursor = dp( a->dCursor ) ;
	P.nDescs = n ; P.nSets = n_sets ; P.kmerLength = kmer_length ;
	std::vector<u64> eo( n_sets ), so( n_sets ) ;
	std::vector<T4Op> opsA( n_sets ), opsB( n_workers ), opsC( n_sets ) ;
	for ( int j = 0 ; j < n_sets ; ++j )
	{
		eo[j] = a->ext[j]->off ;
		so[j] = sets[j]->off ;
		T4Op &x = opsA[j] ;
		memset( &x, 0, sizeof( x ) ) ;
		x.streamOff = eo[j] ;
		x.op = T4_OP_ASSIGN_PREP ;
		x.n = j ;
		x.out = dp( a->dP ) ;
		opsC[j] = x ;
		opsC[j].op = T4_OP_ASSIGN_RECOMPUTE ;
	}
	for ( int b = 0 ; b < n_workers ; ++b )
	{
		T4Op &x = opsB[b] ;
		memset( &x, 0, sizeof( x ) ) ;
		x.streamOff = a->workers[b]->off ;
		x.op = T4_OP_ASSIGN ;
		x.n = b ;
		x.out = dp( a->dP ) ;
	}
	int r = h2d( a->dP, &P, sizeof( P ) ) ;
	if ( !r ) r = dzero( a->dCursor, 256 ) ;
	if ( !r ) r = h2d( dOpsA, opsA.data(), (size_t)n_sets * sizeof( T4Op ) ) ;
	if ( !r ) r = h2d( dOpsB, opsB.data(), (size_t)n_workers * sizeof( T4Op ) ) ;
	if ( !r ) r = h2d( dOpsC, opsC.data(), (size_t)n_sets * sizeof( T4Op ) ) ;
	if ( !r ) r = h2d( dExt, eo.data(), (size_t)n_sets * 8 ) ;
	if ( !r ) r = h2d( dSrc, so.data(), (size_t)n_sets * 8 ) ;
	if ( !r ) r = h2d( dDoff, desc_off, (size_t)( n_sets + 1 ) * 8 ) ;
	if ( !r ) r = launch_ops( T4K_AUX, dOpsA, n_sets, cuda_stream ) ;
	if ( !r ) r = launch_ops( T4K_AUX, dOpsB, n_workers, cuda_stream ) ;
	if ( !r ) r = launch_ops( T4K_AUX, dOpsC, n_sets, cuda_stream ) ;
	a->buf = m.keep() ;
	if ( r )
	{
		T4_API( assign_free )( a ) ;
		return 0 ;
	}
	return a ;
}

static int assign_check( t4_assign *a )
{
	if ( !a || !E.up || a->gen != g_gen )
	{
		set_err( "stale or null t4_assign handle" ) ;
		return T4_E_INVAL ;
	}
	return 0 ;
}

int T4_API( assign_results )( t4_assign *a, int32_t *assign, double *similarity )
{
	int r = assign_check( a ) ;
	if ( r ) return r ;
	r = dsync() ;
	if ( r ) return r ;
	r = T4_API( streams_error )( a->ext.data(), a->nSets ) ;
	if ( r ) return r ;
	r = T4_API( streams_error )( a->workers.data(), (int)a->workers.size() ) ;
	if ( r ) return r ;
	if ( assign && ( r = d2h( assign, a->dAssign, (size_t)a->nDescs * 32 ) ) ) return r ;
	if ( similarity && ( r = d2h( similarity, a->dSim, (size_t)a->nDescs * 8 ) ) ) return r ;
	return 0 ;
}

int T4_API( assign_stats )( t4_assign *a, uint64_t *stats )
{
	int r = assign_check( a ) ;
	if ( r ) return r ;
	r = dsync() ;
	if ( r ) return r ;
	u64 c[4] ;
	r = d2h( c, a->dCursor, sizeof( c ) ) ;
	if ( r ) return r ;
	stats[0] = c[3] ; // reads in the pass (assembled reads)
	stats[1] = c[1] ; // AssignRead calls (identical neighbours share one)
	stats[2] = c[2] ; // reads assigned to a contig
	stats[3] = (u64)a->workers.size() ;
	return 0 ;
}

t4_seqset *T4_API( assign_extended_set )( t4_assign *a, int j )
{
	if ( assign_check( a ) || j < 0 || j >= a->nSets )
		return 0 ;
	return a->ext[j] ;
}

// device pointers of the per-record results for device-side consumers (bench: no host copy inside the timed region)
int T4_API( assign_device_buffers )( t4_assign *a, void **assign, void **similarity )
{
	int r = assign_check( a ) ;
	if ( r ) return r ;
	if ( assign ) *assign = a->dAssign ;
	if ( similarity ) *similarity = a->dSim ;
	return 0 ;
}

// ---- stage-0 candidate extraction against a reference gene set (t4_refscan.h; SURVEY.md 8f-4) ------------------------
struct t4_refset
{
	t4_seqset *set ;                   // the sequences as contigs of one stream, indexed at k
	std::vector<std::string> names ;   // after the de-duplication ("a|b" for identical sequences, SeqSet.hpp:2751-2760)
	std::vector<t4_seqset *> workers ; // scratch-only streams of the scan and annotate launches (created on first use)
	u64 workerPitch ;                  // arena distance between consecutive worker shells (one seqsets_create_impl call)
	char *dbuf ;                       // device: parameter block + op records of the scan launch
	size_t dbufCap ;
	int k ;
	uint32_t gen ;
} ;

static int refset_check( t4_refset *r )
{
	if ( !r || !E.up || r->gen != g_gen )
	{
		set_err( "stale or null t4_refset handle" ) ;
		return T4_E_INVAL ;
	}
	return 0 ;
}

// SeqSet::GetGeneType( name ) == 1 (a D gene), SeqSet.hpp:5076-5100
static bool ref_is_d_gene( const char *name )
{
	if ( name[0] == 'N' && name[1] == 'o' )
		return false ;
	size_t n = strlen( name ) ;
	return n > 4 && name[3] == 'D' && name[4] >= '0' && name[4] <= '9' ;
}

// SeqSet::InputRefFa( file ) with isIMGT == false (SeqSet.hpp:2673-2760, 2864): FASTA records -> cleaned sequences.
// Kept out: non-D genes whose id holds "/OR"; '.' removed; lower case and every character outside A-Z, and every letter
// that is neither ACGT nor N, become 'N' (the reference's lower-case conversion `-= 'a' + 'A'` leaves the range, :2720-2732);
// a sequence seen before is dropped and its name appended to the first one's ("a|b") unless that already contains it.
static int ref_parse_fa( const char *path, std::vector<std::string> &names, std::vector<std::string> &seqs )
{
	FILE *fp = fopen( path, "r" ) ;
	if ( !fp )
	{
		set_err( std::string( "cannot open " ) + path ) ;
		return T4_E_INVAL ;
	}
	std::vector<std::string> ids, raw ;
	{
		std::string line ;
		int ch ;
		bool have = false ;
		auto flush = [&]()
		{
			while ( !line.empty() && ( line.back() == '\r' || line.back() == ' ' || line.back() == '\t' ) )
				line.pop_back() ;
			if ( line.empty() )
				return ;
			if ( line[0] == '>' )
			{
				size_t e = 1 ;
				while ( e < line.size() && line[e] != ' ' && line[e] != '\t' )
					++e ;
				ids.push_back( line.substr( 1, e - 1 ) ) ; // kseq: the id ends at the first white space
				raw.push_back( std::string() ) ;
				have = true ;
			}
			else if ( have )
				raw.back() += line ;
		} ;
		while ( ( ch = fgetc( fp ) ) != EOF )
		{
			if ( ch == '\n' )
			{
				flush() ;
				line.clear() ;
			}
			else
				line.push_back( (char)ch ) ;
		}
		flush() ;
	}
	fclose( fp ) ;
	std::map<std::string, int> existing ;
	for ( size_t r = 0 ; r < ids.size() ; ++r )
	{
		const std::string &id = ids[r] ;
		if ( !ref_is_d_gene( id.c_str() ) )
		{
			size_t i ;
			for ( i = 0 ; i < id.size() ; ++i )
				if ( id[i] == '/' && id.compare( i + 1, 2, "OR" ) == 0 )
					break ;
			if ( i < id.size() )
				continue ;
		}
		std::string cons ;
		for ( size_t i = 0 ; i < raw[r].size() ; ++i )
		{
			char c = raw[r][i] ;
			if ( c == '.' )
				continue ;
			if ( !( c >= 'A' && c <= 'Z' ) )
				c = 'N' ;
			else if ( c != 'A' && c != 'C' && c != 'G' && c != 'T' && c != 'N' )
				c = 'N' ;
			cons.push_back( c ) ;
		}
		std::map<std::string, int>::iterator it = existing.find( cons ) ;
		if ( it != existing.end() )
		{
			std::string &first = names[ it->second ] ;
			if ( first.find( id ) == std::string::npos )
				first += "|" + id ;
			continue ;
		}
		existing[cons] = (int)names.size() ;
		names.push_back( id ) ;
		seqs.push_back( cons ) ;
	}
	return 0 ;
}

void T4_API( refset_free )( t4_refset *r )
{
	if ( !r )
		return ;
	delete r->set ;
	for ( size_t i = 0 ; i < r->workers.size() ; ++i )
		delete r->workers[i] ;
	if ( r->dbuf )
		dfree( r->dbuf ) ;
	delete r ;
}

// `SeqSet refSet( kmer_length ) ; refSet.InputRefFa( fasta_path )` (FastqExtractor.cpp:313-318) on the device
t4_refset *T4_API( refset_create_from_fa )( const char *fasta_path, int kmer_length )
{
	if ( ensure_up() || !fasta_path )
		return 0 ;
	std::vector<std::string> names, seqs ;
	if ( ref_parse_fa( fasta_path, names, seqs ) )
		return 0 ;
	if ( seqs.empty() )
	{
		set_err( "t4_refset_create_from_fa: no sequence in the file" ) ;
		return 0 ;
	}
	t4_refset *r = new t4_refset ;
	r->set = 0 ; r->k = kmer_length ; r->gen = g_gen ; r->workerPitch = 0 ; r->dbuf = 0 ; r->dbufCap = 0 ;
	if ( seqsets_create_impl( 1, kmer_length, 31, 0, &r->set ) )
	{
		delete r ;
		return 0 ;
	}
	const int n = (int)seqs.size() ;
	std::vector<u64> so( n + 1, 0 ), no( n + 1, 0 ) ;
	std::string sp, np ;
	for ( int i = 0 ; i < n ; ++i )
	{
		if ( seqs[i].size() > T4_KEY_B_MASK )
		{
			set_err( "t4_refset_create_from_fa: sequence too long" ) ;
			T4_API( refset_free )( r ) ;
			return 0 ;
		}
		sp += seqs[i] ; np += names[i] ;
		so[i + 1] = sp.size() ; no[i + 1] = np.size() ;
	}
	DevBuf m ;
	T4RefInput *dIn ;
	T4Op *dOp ;
	char *dSp, *dNp ;
	u64 *dSo, *dNo ;
	m.add( dIn, sizeof( T4RefInput ) ) ; m.add( dOp, sizeof( T4Op ) ) ; m.add( dSp, sp.size() + 16 ) ; m.add( dSo, ( n + 1 ) * 8 ) ;
	m.add( dNp, np.size() + 16 ) ; m.add( dNo, ( n + 1 ) * 8 ) ;
	if ( m.alloc() )
	{
		T4_API( refset_free )( r ) ;
		return 0 ;
	}
	T4RefInput in ;
	memset( &in, 0, sizeof( in ) ) ;
	in.seqPool = (u64)(uintptr_t)dSp ; in.seqOff = (u64)(uintptr_t)dSo ;
	in.namePool = (u64)(uintptr_t)dNp ; in.nameOff = (u64)(uintptr_t)dNo ;
	in.n = n ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = r->set->off ;
	op.op = T4_OP_REF_INPUT ;
	op.out = (u64)(uintptr_t)dIn ;
	int rc = h2d( dIn, &in, sizeof( in ) ) ;
	if ( !rc ) rc = h2d( dOp, &op, sizeof( op ) ) ;
	if ( !rc ) rc = h2d( dSp, sp.data(), sp.size() ) ;
	if ( !rc ) rc = h2d( dSo, so.data(), ( n + 1 ) * 8 ) ;
	if ( !rc ) rc = h2d( dNp, np.data(), np.size() ) ;
	if ( !rc ) rc = h2d( dNo, no.data(), ( n + 1 ) * 8 ) ;
	if ( !rc ) rc = launch_ops( T4K_AUX, dOp, 1, 0 ) ;
	if ( !rc ) rc = dsync() ;
	if ( !rc ) rc = d2h( &op, dOp, sizeof( op ) ) ;
	if ( rc || op.ret != n )
	{
		if ( !rc )
			set_err( "t4_refset_create_from_fa: device error " + std::to_string( op.ret ) ) ;
		T4_API( refset_free )( r ) ;
		return 0 ;
	}
	r->names = names ;
	return r ;
}

int T4_API( refset_size )( t4_refset *r ) { return refset_check( r ) ? T4_E_INVAL : (int)r->names.size() ; }
const char *T4_API( refset_name )( t4_refset *r, int i )
{
	if ( refset_check( r ) || i < 0 || i >= (int)r->names.size() )
		return 0 ;
	return r->names[i].c_str() ;
}
// the set behind it (owned by the refset): t4_seqset_get_hits / t4_seqset_get_contig / t4_seqset_index_checksum work on it
t4_seqset *T4_API( refset_seqset )( t4_refset *r ) { return refset_check( r ) ? 0 : r->set ; }
// SeqSet::SetHitLenRequired (FastqExtractor.cpp:455) and SetRadius (SeqSet.hpp:2596)
int T4_API( refset_set_hit_len_required )( t4_refset *r, int l )
{
	int rc = refset_check( r ) ;
	return rc ? rc : put_field( r->set, offsetof( T4Stream, hitLenRequired ), &l, sizeof( int ) ) ;
}
int T4_API( refset_set_radius )( t4_refset *r, int radius )
{
	int rc = refset_check( r ) ;
	return rc ? rc : put_field( r->set, offsetof( T4Stream, radius ), &radius, sizeof( int ) ) ;
}

// At least n scratch-only worker streams (the arena is a bump allocator: shells of an earlier count stay allocated
// until t4_reset).
static int refset_workers( t4_refset *r, int n )
{
	if ( (int)r->workers.size() >= n )
		return 0 ;
	for ( size_t i = 0 ; i < r->workers.size() ; ++i )
		delete r->workers[i] ;
	r->workers.assign( n, (t4_seqset *)0 ) ;
	int rc = seqsets_create_impl( n, r->k, 31, 0, r->workers.data() ) ;
	if ( rc )
		r->workers.clear() ;
	else
		r->workerPitch = n > 1 ? r->workers[1]->off - r->workers[0]->off : sizeof( T4Stream ) ;
	return rc ;
}

// Clears the device error word (error, errorAux) of the first n worker shells, ordered on `stream` before the launch that
// uses them.  A read that fails (e.g. more hits than the per-read scratch holds) fails its own call; the shells are reused
// by every later scan and annotate of the refset, which must not inherit that error.
static int refset_clear_worker_errors( t4_refset *r, int n, void *stream )
{
	char *first = E.A + r->workers[0]->off + offsetof( T4Stream, error ) ;
	static_assert( offsetof( T4Stream, errorAux ) == offsetof( T4Stream, error ) + sizeof( int ), "error word layout" ) ;
#if T4_CUDA
	CK( cudaMemset2DAsync( first, r->workerPitch, 0, 2 * sizeof( int ), n, (cudaStream_t)stream ) ) ;
#else
	(void)stream ;
	for ( int w = 0 ; w < n ; ++w )
		memset( first + (size_t)w * r->workerPitch, 0, 2 * sizeof( int ) ) ;
#endif
	return 0 ;
}

// Host read records: read i is pool[seq_off[i] .. + len[i]).  fn names the entry point in the message.
static int check_records( const char *fn, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len, i64 n )
{
	for ( i64 i = 0 ; i < n ; ++i )
	{
		if ( len[i] > T4_DEV_MAX_READ )
		{
			set_err( std::string( fn ) + ": read longer than the device limit" ) ;
			return T4_E_UNSUPPORTED ;
		}
		if ( len[i] < 0 || seq_off[i] + (u64)len[i] > pool_bytes )
		{
			set_err( std::string( fn ) + ": record outside the pool" ) ;
			return T4_E_INVAL ;
		}
	}
	return 0 ;
}

// Device-pointer form of the scan: `pool`, `seq_off` (u64[n]), `len` (i32[n]), `strand_out` (i8[n]) and `low_out` (u8[n])
// are DEVICE buffers, `ctrl` a device scratch of 64 bytes.  Asynchronous on cuda_stream.
int T4_API( refset_scan_device )( t4_refset *r, const void *pool, const void *seq_off, const void *len, int64_t n, void *strand_out,
	void *low_out, void *ctrl, int n_workers, void *cuda_stream )
{
	int rc = refset_check( r ) ;
	if ( rc ) return rc ;
	if ( n < 0 || !pool || !seq_off || !len || !strand_out || !low_out || !ctrl )
	{
		set_err( "t4_refset_scan: bad argument" ) ;
		return T4_E_INVAL ;
	}
	if ( n_workers <= 0 )
		n_workers = resident_workers() ;
	rc = refset_workers( r, n_workers ) ;
	if ( rc ) return rc ;
	T4ScanParams P ;
	memset( &P, 0, sizeof( P ) ) ;
	P.pool = (u64)(uintptr_t)pool ; P.seqOff = (u64)(uintptr_t)seq_off ; P.len = (u64)(uintptr_t)len ;
	P.strandOut = (u64)(uintptr_t)strand_out ; P.lowOut = (u64)(uintptr_t)low_out ; P.cursor = (u64)(uintptr_t)ctrl ;
	P.setOff = r->set->off ;
	P.n = n ;
	// parameter block + op records: a device buffer of the refset (the launch reads them until it ends)
	const size_t need = 256 + (size_t)n_workers * sizeof( T4Op ) ;
	if ( need > r->dbufCap )
	{
		if ( r->dbuf )
			dfree( r->dbuf ) ;
		r->dbuf = 0 ; r->dbufCap = 0 ;
		void *q = 0 ;
		rc = dmalloc( &q, need ) ;
		if ( rc ) return rc ;
		r->dbuf = (char *)q ;
		r->dbufCap = need ;
	}
	std::vector<T4Op> ops( n_workers ) ;
	for ( int b = 0 ; b < n_workers ; ++b )
	{
		T4Op &x = ops[b] ;
		memset( &x, 0, sizeof( x ) ) ;
		x.streamOff = r->workers[b]->off ;
		x.op = T4_OP_REF_SCAN ;
		x.n = b ;
		x.out = (u64)(uintptr_t)r->dbuf ;
	}
	if ( ( rc = h2d_async( r->dbuf, &P, sizeof( P ), cuda_stream ) ) || ( rc = h2d_async( r->dbuf + 256, ops.data(), (size_t)n_workers * sizeof( T4Op ), cuda_stream ) )
		|| ( rc = dzero( ctrl, 32, cuda_stream ) ) || ( rc = refset_clear_worker_errors( r, n_workers, cuda_stream ) ) )
		return rc ;
	return launch_ops( T4K_AUX, (T4Op *)( r->dbuf + 256 ), n_workers, cuda_stream ) ;
}

// Host form: for every read IsLowComplexity( read ) and refSet->HasHitInSet( read, 0 ) -- fastq-extractor keeps a read
// (pair) when `!low && strand != 0` holds for it (or its mate), FastqExtractor.cpp:129-134, 211-219.
// stats (may be NULL): [0] reads with a hit, [1] low-complexity reads.
int T4_API( refset_scan )( t4_refset *r, const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len, int64_t n,
	int8_t *strand_out, uint8_t *low_complexity_out, uint64_t *stats )
{
	int rc = refset_check( r ) ;
	if ( rc ) return rc ;
	if ( n < 0 || !read_pool || !seq_off || !len )
	{
		set_err( "t4_refset_scan: bad argument" ) ;
		return T4_E_INVAL ;
	}
	rc = check_records( "t4_refset_scan", pool_bytes, seq_off, len, n ) ;
	if ( rc || n == 0 )
		return rc ;
	DevBuf m ;
	char *dPool ;
	u64 *dOff, *dCtrl ;
	int32_t *dLen ;
	int8_t *dStr ;
	uint8_t *dLow ;
	m.add( dPool, pool_bytes + 16 ) ; m.add( dOff, (size_t)n * 8 ) ; m.add( dLen, (size_t)n * 4 ) ; m.add( dStr, (size_t)n ) ; m.add( dLow, (size_t)n ) ;
	m.add( dCtrl, 256 ) ;
	rc = m.alloc() ;
	if ( !rc ) rc = h2d( dPool, read_pool, pool_bytes ) ;
	if ( !rc ) rc = h2d( dOff, seq_off, (size_t)n * 8 ) ;
	if ( !rc ) rc = h2d( dLen, len, (size_t)n * 4 ) ;
	const int nw = resident_workers() ;
	if ( !rc ) rc = T4_API( refset_scan_device )( r, dPool, dOff, dLen, n, dStr, dLow, dCtrl, nw, 0 ) ;
	if ( !rc ) rc = dsync() ;
	if ( !rc ) rc = T4_API( streams_error )( r->workers.data(), nw ) ;
	if ( !rc && strand_out ) rc = d2h( strand_out, dStr, (size_t)n ) ;
	if ( !rc && low_complexity_out ) rc = d2h( low_complexity_out, dLow, (size_t)n ) ;
	if ( !rc && stats )
	{
		u64 c[4] ;
		rc = d2h( c, dCtrl, sizeof( c ) ) ;
		stats[0] = c[1] ; stats[1] = c[2] ;
	}
	return rc ;
}

// SeqSet::GetOverlapsFromRead( read, 0, -1, 0, false, overlaps ) on the reference gene set (the call AnnotateRead makes per
// read, SeqSet.hpp:6050): overlaps as int32[8] = {seqIdx, readStart, readEnd, seqStart, seqEnd, strand, matchCnt, indelCnt}
// plus similarity[i], in the reference's order.  Returns the overlap count, -1 for a read shorter than k.
// Verified on the GPU against the reference (see t4_annot.h).
int T4_API( refset_get_overlaps )( t4_refset *r, const char *read, int32_t *overlaps, double *similarity, int cap )
{
	int rc = refset_check( r ) ;
	if ( rc ) return rc ;
	int len ;
	rc = read_ok( read, &len ) ;
	if ( rc ) return rc ;
	if ( cap < 0 || ( cap > 0 && ( !overlaps || !similarity ) ) )
		return T4_E_INVAL ;
	T4Stream st ;
	rc = get_stream( r->set, &st ) ;
	if ( rc ) return rc ;
	if ( st.error ) // raised by something other than an earlier get_overlaps (those clear it below): still reported
	{
		set_err( "t4_refset_get_overlaps: the gene set carries device error " + std::to_string( st.error ) + " aux " + std::to_string( st.errorAux ) ) ;
		return st.error ;
	}
	const int hMax = 1 << 16 ;
	const size_t sb = t4_annot_scratch_bytes( hMax, st.nomatchGapLimit, T4_DEV_MAX_READ ) ;
	DevBuf m ;
	T4Op *dOp ;
	T4RefOvlParams *dPar ;
	char *dRead, *dOut, *dScr ;
	m.add( dOp, sizeof( T4Op ) ) ; m.add( dPar, sizeof( T4RefOvlParams ) ) ; m.add( dRead, (size_t)len + 16 ) ; m.add( dOut, (size_t)cap * 40 + 64 ) ;
	m.add( dScr, sb ) ;
	rc = m.alloc() ;
	if ( rc ) return rc ;
	T4RefOvlParams P ;
	memset( &P, 0, sizeof( P ) ) ;
	P.scratch = (u64)(uintptr_t)dScr ;
	P.scratchBytes = sb ;
	P.hMax = hMax ;
	T4Op op ;
	memset( &op, 0, sizeof( op ) ) ;
	op.streamOff = r->set->off ;
	op.op = T4_OP_REF_OVERLAPS ;
	op.read = (u64)(uintptr_t)dRead ;
	op.len = len ;
	op.out = (u64)(uintptr_t)dOut ;
	op.out2 = (u64)(uintptr_t)dPar ;
	op.outCap = cap ;
	rc = h2d( dOp, &op, sizeof( op ) ) ;
	if ( !rc ) rc = h2d( dPar, &P, sizeof( P ) ) ;
	if ( !rc ) rc = h2d( dRead, read, (size_t)len + 1 ) ;
	if ( !rc ) rc = launch_ops( T4K_ANNOT, dOp, 1, 0 ) ;
	if ( !rc ) rc = dsync() ;
	if ( !rc ) rc = d2h( &op, dOp, sizeof( op ) ) ;
	int n = op.ret ;
	if ( !rc && n > 0 )
	{
		const int k = n < cap ? n : cap ;
		rc = d2h( overlaps, dOut, (size_t)k * 32 ) ;
		if ( !rc ) rc = d2h( similarity, dOut + (size_t)cap * 32, (size_t)k * 8 ) ;
	}
	if ( rc ) return rc ;
	if ( n < T4_E_BASE )
	{
		// the op runs on the set's own stream, so the error this read raised sits in the set's error word: report it, then
		// clear the word so that the next read is answered on its own
		rc = get_stream( r->set, &st ) ;
		if ( rc ) return rc ;
		set_err( "t4_refset_get_overlaps: device error " + std::to_string( n ) + " aux " + std::to_string( st.errorAux ) ) ;
		const int clear[2] = { 0, 0 } ;
		rc = put_field( r->set, offsetof( T4Stream, error ), clear, sizeof( clear ) ) ;
		if ( rc ) return rc ;
	}
	return n ;
}

// SeqSet::AnnotateRead( read, 0, geneOverlap, NULL, NULL ) for every read (the rough annotation of the stage-1 driver,
// main.cpp:1084-1120; SeqSet.hpp:6016-6340): gene_overlaps[i][t][8] for t = V, D, J, C = {seqIdx (-1: none), readStart,
// readEnd, seqStart, seqEnd, strand, matchCnt, indelCnt}, similarity[i][t].  Host buffers.
// Verified on the GPU against the reference (see t4_annot.h).
int T4_API( refset_annotate )( t4_refset *r, const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len, int64_t n,
	int32_t *gene_overlaps, double *similarity )
{
	int rc = refset_check( r ) ;
	if ( rc ) return rc ;
	if ( n < 0 || !read_pool || !seq_off || !len || !gene_overlaps || !similarity )
	{
		set_err( "t4_refset_annotate: bad argument" ) ;
		return T4_E_INVAL ;
	}
	rc = check_records( "t4_refset_annotate", pool_bytes, seq_off, len, n ) ;
	if ( rc || n == 0 )
		return rc ;
	T4Stream st ;
	rc = get_stream( r->set, &st ) ;
	if ( rc ) return rc ;
	int nw = resident_workers() ;
	if ( (i64)nw > n )
		nw = (int)n ;
	rc = refset_workers( r, nw ) ;
	if ( rc ) return rc ;
	const int hMax = 1 << 16 ; // hits of one read (contig) a worker has serial work space for: 16 MB per worker
	const size_t stride = ( t4_annot_scratch_bytes( hMax, st.nomatchGapLimit, T4_DEV_MAX_READ, st.nSeqs ) + 255 ) & ~(size_t)255 ;
	DevBuf m ;
	T4AnnotParams *dPar ;
	T4Op *dOps ;
	char *dPool, *dScr ;
	u64 *dOff, *dCtrl ;
	int32_t *dLen, *dOut ;
	double *dSim ;
	m.add( dPar, sizeof( T4AnnotParams ) ) ; m.add( dOps, (size_t)nw * sizeof( T4Op ) ) ; m.add( dPool, pool_bytes + 16 ) ; m.add( dOff, (size_t)n * 8 ) ;
	m.add( dLen, (size_t)n * 4 ) ; m.add( dOut, (size_t)n * 4 * 8 * 4 ) ; m.add( dSim, (size_t)n * 4 * 8 ) ; m.add( dCtrl, 256 ) ;
	m.add( dScr, stride * (size_t)nw ) ;
	rc = m.alloc() ;
	if ( rc ) return rc ;
	T4AnnotParams P ;
	memset( &P, 0, sizeof( P ) ) ;
	P.pool = (u64)(uintptr_t)dPool ; P.seqOff = (u64)(uintptr_t)dOff ; P.len = (u64)(uintptr_t)dLen ;
	P.out = (u64)(uintptr_t)dOut ; P.sim = (u64)(uintptr_t)dSim ; P.cursor = (u64)(uintptr_t)dCtrl ;
	P.setOff = r->set->off ;
	P.scratch = (u64)(uintptr_t)dScr ; P.scratchStride = stride ;
	P.n = n ; P.hMax = hMax ;
	std::vector<T4Op> ops( nw ) ;
	for ( int w = 0 ; w < nw ; ++w )
	{
		memset( &ops[w], 0, sizeof( T4Op ) ) ;
		ops[w].streamOff = r->workers[w]->off ;
		ops[w].op = T4_OP_REF_ANNOTATE ;
		ops[w].n = w ;
		ops[w].out = (u64)(uintptr_t)dPar ;
	}
	rc = h2d( dPar, &P, sizeof( P ) ) ;
	if ( !rc ) rc = h2d( dOps, ops.data(), (size_t)nw * sizeof( T4Op ) ) ;
	if ( !rc ) rc = h2d( dPool, read_pool, pool_bytes ) ;
	if ( !rc ) rc = h2d( dOff, seq_off, (size_t)n * 8 ) ;
	if ( !rc ) rc = h2d( dLen, len, (size_t)n * 4 ) ;
	if ( !rc ) rc = dzero( dCtrl, 64 ) ;
	if ( !rc ) rc = refset_clear_worker_errors( r, nw, 0 ) ;
	if ( !rc ) rc = launch_ops( T4K_ANNOT, dOps, nw, 0 ) ;
	if ( !rc ) rc = dsync() ;
	if ( !rc ) rc = T4_API( streams_error )( r->workers.data(), nw ) ;
	if ( !rc ) rc = d2h( gene_overlaps, dOut, (size_t)n * 4 * 8 * 4 ) ;
	if ( !rc ) rc = d2h( similarity, dSim, (size_t)n * 4 * 8 ) ;
	return rc ;
}

// `std::sort( sortedReads.begin(), sortedReads.end() )` of the stage-1 driver (main.cpp:1078; _sortRead::operator<, :103-125):
// order[j] = index of the record that comes j-th.  Host buffers; record i: read_pool[seq_off[i] .. + len[i]), its id
// id_pool[id_off[i] .. id_off[i + 1]), its count statistics.  Verified on the GPU (t4_readsort.h).
} // extern "C" (C++ helpers of the two sort entry points)
static T4SortRec &sort_rec_base( T4SortRec &r ) { return r ; }
static T4SortRec &sort_rec_base( T4SortRecBc &r ) { return r.r ; }

// The merge sort of t4_sort_reads / t4_sort_reads_barcode over records the caller filled except for the read and id
// fields (checked and set here); `kernel` is the merge pass of the record type.
template <class Rec, class K> static int sort_records( const char *fn, K kernel, std::vector<Rec> &recs, const char *read_pool,
	size_t pool_bytes, const uint64_t *seq_off, const int32_t *len, const char *id_pool, size_t id_pool_bytes, const uint64_t *id_off,
	int64_t n, int64_t *order )
{
	std::vector<i64> idx( (size_t)n ) ;
	for ( i64 i = 0 ; i < n ; ++i )
	{
		if ( len[i] < 0 || seq_off[i] + (u64)len[i] > pool_bytes || id_off[i + 1] < id_off[i] || id_off[i + 1] > id_pool_bytes )
		{
			set_err( std::string( fn ) + ": record outside its pool" ) ;
			return T4_E_INVAL ;
		}
		T4SortRec &r = sort_rec_base( recs[(size_t)i] ) ;
		r.len = len[i] ;
		r.readOff = seq_off[i] ; r.idOff = id_off[i] ; r.idLen = (int32_t)( id_off[i + 1] - id_off[i] ) ; r.pad = 0 ;
		idx[(size_t)i] = i ;
	}
	DevBuf m ;
	Rec *dRec ;
	char *dPool, *dId ;
	i64 *from, *to ;
	m.add( dRec, (size_t)n * sizeof( Rec ) ) ; m.add( dPool, pool_bytes + 16 ) ; m.add( dId, id_pool_bytes + 16 ) ; m.add( from, (size_t)n * 8 ) ;
	m.add( to, (size_t)n * 8 ) ;
	int rc = m.alloc() ;
	if ( !rc ) rc = h2d( dRec, recs.data(), (size_t)n * sizeof( Rec ) ) ;
	if ( !rc ) rc = h2d( dPool, read_pool, pool_bytes ) ;
	if ( !rc ) rc = h2d( dId, id_pool, id_pool_bytes ) ;
	if ( !rc ) rc = h2d( from, idx.data(), (size_t)n * 8 ) ;
	T4SortParams P ;
	memset( &P, 0, sizeof( P ) ) ;
	P.recs = (u64)(uintptr_t)dRec ; P.pool = (u64)(uintptr_t)dPool ; P.idPool = (u64)(uintptr_t)dId ;
	P.n = n ;
	for ( i64 w = 1 ; !rc && w < n ; w *= 2 )
	{
		P.src = (u64)(uintptr_t)from ; P.dst = (u64)(uintptr_t)to ; P.width = w ;
		rc = launch_items( kernel, P, n, 256 ) ;
		i64 *t = from ; from = to ; to = t ;
	}
	if ( !rc ) rc = dsync() ;
	if ( !rc ) rc = d2h( order, from, (size_t)n * 8 ) ;
	return rc ;
}
extern "C" {

int T4_API( sort_reads )( const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len, const char *id_pool,
	size_t id_pool_bytes, const uint64_t *id_off, const int32_t *min_cnt, const int32_t *median_cnt, const float *avg_cnt, int64_t n,
	int64_t *order )
{
	int rc = ensure_up() ;
	if ( rc ) return rc ;
	if ( n < 0 || !read_pool || !seq_off || !len || !id_pool || !id_off || !min_cnt || !median_cnt || !avg_cnt || !order )
	{
		set_err( "t4_sort_reads: bad argument" ) ;
		return T4_E_INVAL ;
	}
	if ( n == 0 )
		return 0 ;
	std::vector<T4SortRec> recs( (size_t)n ) ;
	for ( i64 i = 0 ; i < n ; ++i )
	{
		T4SortRec &r = recs[(size_t)i] ;
		r.minCnt = min_cnt[i] ; r.medianCnt = median_cnt[i] ; r.avgCnt = avg_cnt[i] ;
	}
	return sort_records( "t4_sort_reads", T4_KERNEL( t4_readsort_kernel, t4_sort_merge_one<T4SortRec> ), recs, read_pool, pool_bytes, seq_off,
		len, id_pool, id_pool_bytes, id_off, n, order ) ;
}

// `CompReadWithBarcode` order of a --barcode run (main.cpp:128-136): t4_sort_reads' records plus barcode[i] (>= 0) and
// barcode_min_cnt[i].  One sort in this order, after the per-cell counts are known, is what the driver's two sorts
// produce together (main.cpp:1126 while every barcodeMinCnt is still 0, i.e. grouped by barcode; then each barcode
// group again at :1183-1192).  Host buffers; negative barcodes give T4_E_INVAL.  Verified on the GPU (t4_readsort.h).
int T4_API( sort_reads_barcode )( const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len, const char *id_pool,
	size_t id_pool_bytes, const uint64_t *id_off, const int32_t *min_cnt, const int32_t *median_cnt, const float *avg_cnt,
	const int32_t *barcode, const int32_t *barcode_min_cnt, int64_t n, int64_t *order )
{
	int rc = ensure_up() ;
	if ( rc ) return rc ;
	if ( n < 0 || !read_pool || !seq_off || !len || !id_pool || !id_off || !min_cnt || !median_cnt || !avg_cnt || !barcode
		|| !barcode_min_cnt || !order )
	{
		set_err( "t4_sort_reads_barcode: bad argument" ) ;
		return T4_E_INVAL ;
	}
	std::vector<T4SortRecBc> recs( (size_t)n ) ;
	for ( i64 i = 0 ; i < n ; ++i )
	{
		if ( barcode[i] < 0 )
		{
			set_err( "t4_sort_reads_barcode: negative barcode (CompReadWithBarcode is an order only on barcodes >= 0)" ) ;
			return T4_E_INVAL ;
		}
		T4SortRecBc &r = recs[(size_t)i] ;
		r.r.minCnt = min_cnt[i] ; r.r.medianCnt = median_cnt[i] ; r.r.avgCnt = avg_cnt[i] ;
		r.barcode = barcode[i] ; r.barcodeMinCnt = barcode_min_cnt[i] ;
	}
	if ( n == 0 )
		return 0 ;
	return sort_records( "t4_sort_reads_barcode", T4_KERNEL( t4_readsort_bc_kernel, t4_sort_merge_one<T4SortRecBc> ), recs, read_pool,
		pool_bytes, seq_off, len, id_pool, id_pool_bytes, id_off, n, order ) ;
}

// AlignAlgo::IsMateOverlap for n (first, second) read pairs of one pool (ProcessRead, main.cpp:264, 291): overlap_size[i] =
// the return value (-1: no unambiguous overlap), offset[i] / best_match_cnt[i] the two reference outputs.  Host buffers.
// Verified on the GPU against the reference (t4_readsort.h).
int T4_API( mate_overlap_batch )( const char *read_pool, size_t pool_bytes, const uint64_t *f_off, const int32_t *f_len, const uint64_t *s_off,
	const int32_t *s_len, const int32_t *min_overlap, const uint8_t *check_tandem, int64_t n, int32_t *overlap_size, int32_t *offset,
	int32_t *best_match_cnt )
{
	int rc = ensure_up() ;
	if ( rc ) return rc ;
	if ( n < 0 || !read_pool || !f_off || !f_len || !s_off || !s_len || !min_overlap || !check_tandem || !overlap_size || !offset || !best_match_cnt )
	{
		set_err( "t4_mate_overlap_batch: bad argument" ) ;
		return T4_E_INVAL ;
	}
	for ( i64 i = 0 ; i < n ; ++i )
		if ( f_len[i] < 0 || s_len[i] < 0 || f_off[i] + (u64)f_len[i] > pool_bytes || s_off[i] + (u64)s_len[i] > pool_bytes )
		{
			set_err( "t4_mate_overlap_batch: record outside the pool" ) ;
			return T4_E_INVAL ;
		}
	if ( n == 0 )
		return 0 ;
	DevBuf m ;
	char *dPool ;
	u64 *dFo, *dSo ;
	int32_t *dFl, *dSl, *dMo, *dOs, *dOf, *dBm ;
	uint8_t *dCt ;
	m.add( dPool, pool_bytes + 16 ) ; m.add( dFo, (size_t)n * 8 ) ; m.add( dSo, (size_t)n * 8 ) ; m.add( dFl, (size_t)n * 4 ) ; m.add( dSl, (size_t)n * 4 ) ;
	m.add( dMo, (size_t)n * 4 ) ; m.add( dCt, (size_t)n ) ; m.add( dOs, (size_t)n * 4 ) ; m.add( dOf, (size_t)n * 4 ) ; m.add( dBm, (size_t)n * 4 ) ;
	rc = m.alloc() ;
	if ( !rc ) rc = h2d( dPool, read_pool, pool_bytes ) ;
	if ( !rc ) rc = h2d( dFo, f_off, (size_t)n * 8 ) ;
	if ( !rc ) rc = h2d( dSo, s_off, (size_t)n * 8 ) ;
	if ( !rc ) rc = h2d( dFl, f_len, (size_t)n * 4 ) ;
	if ( !rc ) rc = h2d( dSl, s_len, (size_t)n * 4 ) ;
	if ( !rc ) rc = h2d( dMo, min_overlap, (size_t)n * 4 ) ;
	if ( !rc ) rc = h2d( dCt, check_tandem, (size_t)n ) ;
	T4MateParams P ;
	memset( &P, 0, sizeof( P ) ) ;
	auto dp = []( const void *q ) { return (u64)(uintptr_t)q ; } ;
	P.pool = dp( dPool ) ; P.fOff = dp( dFo ) ; P.sOff = dp( dSo ) ; P.fLen = dp( dFl ) ; P.sLen = dp( dSl ) ; P.minOverlap = dp( dMo ) ;
	P.checkTandem = dp( dCt ) ; P.overlapSize = dp( dOs ) ; P.offset = dp( dOf ) ; P.bestMatchCnt = dp( dBm ) ;
	P.n = n ;
	if ( !rc ) rc = launch_items( T4_KERNEL( t4_mate_overlap_kernel, t4_mate_overlap_one ), P, n, 128 ) ;
	if ( !rc ) rc = dsync() ;
	if ( !rc ) rc = d2h( overlap_size, dOs, (size_t)n * 4 ) ;
	if ( !rc ) rc = d2h( offset, dOf, (size_t)n * 4 ) ;
	if ( !rc ) rc = d2h( best_match_cnt, dBm, (size_t)n * 4 ) ;
	return rc ;
}

// Test hook (host only, no device): SeqSet::LongestIncreasingSubsequence (SeqSet.hpp:342-474) as the stage-0 scan runs it --
// hits (a[i], b[i]) sorted by b; the chain goes to out_a / out_b (room for n); returns its length.
int T4_API( test_lis )( const int32_t *a, const int32_t *b, int n, int32_t *out_a, int32_t *out_b )
{
	if ( n <= 0 || !a || !b || !out_a || !out_b )
		return 0 ;
	std::vector<int> top( n ), link( n ) ;
	return t4_lis( a, b, n, top.data(), link.data(), out_a, out_b ) ;
}

// ---- canonical k-mer counts + per-read statistics (t4_kcount.h; SURVEY.md 8f-3) ------------------------------------
// B == NULL: the global table; else the per-cell pass over the barcodes of [B->lo, B->lo + 2^21)
static int kc_launch( const T4KcParams &P, int stats, void *stream, const T4KcBarcode *B = NULL )
{
#if T4_CUDA
	CK( cudaMemsetAsync( (void *)(uintptr_t)P.ctrl, 0, 8, (cudaStream_t)stream ) ) ; // the read cursor
	if ( B ) // 40 warps per SM (21 KB of shared memory per CTA)
		t4_kcount_bc_kernel<<<E.sms * 10, T4_MAX_NT, 0, (cudaStream_t)stream>>>( P, stats, *B ) ;
	else
		t4_kcount_kernel<<<E.sms * 10, T4_MAX_NT, 0, (cudaStream_t)stream>>>( P, stats ) ;
	CK( cudaGetLastError() ) ;
#else
	*(u64 *)(uintptr_t)P.ctrl = 0 ;
	T4KcSmem *sm = new T4KcSmem ;
	T4KcCtx cx ;
	cx.sm = sm ; cx.tid = 0 ; cx.nt = 1 ;
	const T4KcBarcode none = { 0, 0, 0 } ;
	if ( B && stats )
		kc_stats_body<true>( cx, P, *B ) ;
	else if ( B )
		kc_count_body<true>( cx, P, *B ) ;
	else if ( stats )
		kc_stats_body<false>( cx, P, none ) ;
	else
		kc_count_body<false>( cx, P, none ) ;
	delete sm ;
#endif
	return 0 ;
}

// Device-pointer form: `pool`, `seq_off` (u64[n]), `len` (i32[n]) and the three outputs are DEVICE buffers (e.g. torch
// tensors), `table` is a caller-provided device buffer of t4_kmer_count_table_bytes() bytes.  Asynchronous on cuda_stream.
size_t T4_API( kmer_count_table_bytes )( int64_t n_kmer_instances )
{
	u64 cap = 1024 ;
	while ( cap < 2 * (u64)( n_kmer_instances > 0 ? n_kmer_instances : 0 ) )
		cap <<= 1 ;
	return (size_t)( cap * 12 + 256 ) ;
}

int T4_API( kmer_count_stats_device )( const void *pool, const void *qual, const void *seq_off, const void *len, int64_t n, int kmer_length,
	void *table, size_t table_bytes, void *min_cnt, void *median_cnt, void *avg_cnt, void *new_len, void *cuda_stream )
{
	int r = ensure_up() ;
	if ( r ) return r ;
	if ( n < 0 || kmer_length < 2 || kmer_length > 31 || table_bytes < 1024 * 12 + 256 )
	{
		set_err( "t4_kmer_count_stats: bad argument" ) ;
		return T4_E_INVAL ;
	}
	u64 cap = 1024 ;
	while ( cap * 2 * 12 + 256 <= table_bytes )
		cap <<= 1 ;
	T4KcParams P ;
	memset( &P, 0, sizeof( P ) ) ;
	char *t = (char *)table ;
	P.keys = (u64)(uintptr_t)t ;
	P.counts = (u64)(uintptr_t)( t + cap * 8 ) ;
	P.ctrl = (u64)(uintptr_t)( t + cap * 12 ) ;
	P.cap = cap ;
	P.pool = (u64)(uintptr_t)pool ;
	P.seqOff = (u64)(uintptr_t)seq_off ;
	P.len = (u64)(uintptr_t)len ;
	P.minCnt = (u64)(uintptr_t)min_cnt ;
	P.medianCnt = (u64)(uintptr_t)median_cnt ;
	P.avgCnt = (u64)(uintptr_t)avg_cnt ;
	P.qual = (u64)(uintptr_t)qual ;
	P.newLen = (u64)(uintptr_t)new_len ;
	P.n = n ;
	P.k = kmer_length ;
	r = dzero( table, cap * 12 + 64, cuda_stream ) ;
	if ( !r ) r = kc_launch( P, 0, cuda_stream ) ;
	if ( !r ) r = kc_launch( P, 1, cuda_stream ) ;
	return r ;
}

// Totals of the last call on this table (synchronises): stats[0] k-mers counted, [1] distinct k-mers, [2] table slots,
// [3] 1 if the table overflowed (results invalid).
int T4_API( kmer_count_table_stats )( const void *table, size_t table_bytes, uint64_t *stats )
{
	u64 cap = 1024 ;
	while ( cap * 2 * 12 + 256 <= table_bytes )
		cap <<= 1 ;
	int r = dsync() ;
	if ( r ) return r ;
	u64 c[4] ;
	r = d2h( c, (const char *)table + cap * 12, sizeof( c ) ) ;
	if ( r ) return r ;
	stats[0] = c[1] ; stats[1] = c[2] ; stats[2] = cap ; stats[3] = c[3] ;
	return 0 ;
}

// Host form: KmerCount( kmer_length ).AddCount( read ) for every read, then GetCountStatsAndTrim( read, qual, ... ) for
// every read (main.cpp:404-440, 981-1010; qual_pool == NULL: no trimming).  Reads longer than T4_MAX_READ_LEN are not supported (T4_E_UNSUPPORTED).
int T4_API( kmer_count_stats )( const char *read_pool, const char *qual_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len,
	int64_t n, int kmer_length, int32_t *min_cnt, int32_t *median_cnt, float *avg_cnt, int32_t *new_len )
{
	int r = ensure_up() ;
	if ( r ) return r ;
	if ( n < 0 || !read_pool || !seq_off || !len || kmer_length < 2 || kmer_length > 31 )
	{
		set_err( "t4_kmer_count_stats: bad argument" ) ;
		return T4_E_INVAL ;
	}
	r = check_records( "t4_kmer_count_stats", pool_bytes, seq_off, len, n ) ;
	if ( r || n == 0 )
		return r ;
	u64 inst = 0 ;
	for ( i64 i = 0 ; i < n ; ++i )
		if ( len[i] >= kmer_length )
			inst += (u64)( len[i] - kmer_length + 1 ) ;
	const size_t tb = T4_API( kmer_count_table_bytes )( (int64_t)inst ) ;
	DevBuf m ;
	char *dPool, *dQual, *dTab ;
	u64 *dOff ;
	int32_t *dLen, *dMin, *dMed, *dNew ;
	float *dAvg ;
	m.add( dPool, pool_bytes + 16 ) ; m.add( dQual, qual_pool ? pool_bytes + 16 : 0 ) ; m.add( dOff, (size_t)n * 8 ) ; m.add( dLen, (size_t)n * 4 ) ;
	m.add( dMin, (size_t)n * 4 ) ; m.add( dMed, (size_t)n * 4 ) ; m.add( dAvg, (size_t)n * 4 ) ; m.add( dNew, (size_t)n * 4 ) ; m.add( dTab, tb ) ;
	r = m.alloc() ;
	if ( !r ) r = h2d( dPool, read_pool, pool_bytes ) ;
	if ( !r && qual_pool ) r = h2d( dQual, qual_pool, pool_bytes ) ;
	if ( !r ) r = h2d( dOff, seq_off, (size_t)n * 8 ) ;
	if ( !r ) r = h2d( dLen, len, (size_t)n * 4 ) ;
	if ( !r ) r = T4_API( kmer_count_stats_device )( dPool, qual_pool ? dQual : 0, dOff, dLen, n, kmer_length, dTab, tb, dMin, dMed, dAvg, dNew, 0 ) ;
	u64 st[4] = { 0, 0, 0, 0 } ;
	if ( !r ) r = T4_API( kmer_count_table_stats )( dTab, tb, st ) ;
	if ( !r && st[3] )
	{
		set_err( "t4_kmer_count_stats: count table overflow" ) ;
		r = T4_E_INTERNAL ;
	}
	if ( !r && min_cnt ) r = d2h( min_cnt, dMin, (size_t)n * 4 ) ;
	if ( !r && median_cnt ) r = d2h( median_cnt, dMed, (size_t)n * 4 ) ;
	if ( !r && avg_cnt ) r = d2h( avg_cnt, dAvg, (size_t)n * 4 ) ;
	if ( !r && new_len ) r = d2h( new_len, dNew, (size_t)n * 4 ) ;
	return r ;
}

// The per-cell passes of the device form: one count + statistics launch pair per barcode range of 2^21 ids in `ranges`
// (range j = barcodes [j << 21, (j + 1) << 21)).  The table is cleared before each pass; ctrl[1..3] add up over the passes.
static int bc_kc_passes( T4KcParams &P, const void *barcode, int barcode_max, const std::vector<int> &ranges, void *stream )
{
	int r = 0 ;
	T4KcBarcode B ;
	B.barcode = (u64)(uintptr_t)barcode ;
	B.max = barcode_max ;
	for ( size_t j = 0 ; !r && j < ranges.size() ; ++j )
	{
		B.lo = ranges[j] << T4_KC_BC_BITS ;
		r = dzero( (void *)(uintptr_t)P.keys, P.cap * 12, stream ) ; // keys and counts; ctrl keeps the totals
		if ( !r ) r = kc_launch( P, 0, stream, &B ) ;
		if ( !r ) r = kc_launch( P, 1, stream, &B ) ;
	}
	return r ;
}

static void kc_params( T4KcParams &P, void *table, size_t table_bytes, const void *pool, const void *seq_off, const void *len, int64_t n,
	int k, void *min_cnt, void *median_cnt, void *avg_cnt )
{
	u64 cap = 1024 ;
	while ( cap * 2 * 12 + 256 <= table_bytes )
		cap <<= 1 ;
	memset( &P, 0, sizeof( P ) ) ;
	char *t = (char *)table ;
	P.keys = (u64)(uintptr_t)t ;
	P.counts = (u64)(uintptr_t)( t + cap * 8 ) ;
	P.ctrl = (u64)(uintptr_t)( t + cap * 12 ) ;
	P.cap = cap ;
	P.pool = (u64)(uintptr_t)pool ;
	P.seqOff = (u64)(uintptr_t)seq_off ;
	P.len = (u64)(uintptr_t)len ;
	P.minCnt = (u64)(uintptr_t)min_cnt ;
	P.medianCnt = (u64)(uintptr_t)median_cnt ;
	P.avgCnt = (u64)(uintptr_t)avg_cnt ;
	P.n = n ;
	P.k = k ;
}

// Device-pointer form of the per-cell statistics: `pool`, `seq_off` (u64[n]), `len` (i32[n]), `barcode` (i32[n], every
// id in [0, barcode_max]) and the outputs are DEVICE buffers, `table` a device buffer of t4_kmer_count_table_bytes()
// bytes.  Runs one pass per 2^21 barcode ids up to barcode_max.  Asynchronous on cuda_stream; t4_kmer_count_table_stats
// then reports the totals and whether the results are invalid (stats[3] = 1 table overflow, 2 a barcode outside
// [0, barcode_max]).
int T4_API( barcode_kmer_count_stats_device )( const void *pool, const void *seq_off, const void *len, const void *barcode, int64_t n,
	int32_t barcode_max, int kmer_length, void *table, size_t table_bytes, void *min_cnt, void *median_cnt, void *avg_cnt, void *cuda_stream )
{
	int r = ensure_up() ;
	if ( r ) return r ;
	if ( n < 0 || barcode_max < 0 || kmer_length < 2 || kmer_length > 21 || table_bytes < 1024 * 12 + 256 )
	{
		set_err( "t4_barcode_kmer_count_stats: bad argument" ) ;
		return T4_E_INVAL ;
	}
	T4KcParams P ;
	kc_params( P, table, table_bytes, pool, seq_off, len, n, kmer_length, min_cnt, median_cnt, avg_cnt ) ;
	std::vector<int> ranges ;
	for ( int j = 0 ; j <= ( barcode_max >> T4_KC_BC_BITS ) ; ++j )
		ranges.push_back( j ) ;
	r = dzero( table, P.cap * 12 + 64, cuda_stream ) ;
	if ( !r ) r = bc_kc_passes( P, barcode, barcode_max, ranges, cuda_stream ) ;
	return r ;
}

// The barcode-wise statistics of a --barcode run (main.cpp:1128-1180, BarcodeKmerCount_Thread :569-604): for every
// barcode, KmerCount( kmer_length ) over the reads of that barcode only, then GetCountStatsAndTrim( read, NULL, ... )
// into bc_min_cnt / bc_median_cnt / bc_avg_cnt.  Reads may come in any order.  Host buffers; barcode ids in [0, 2^31);
// negative ones and kmer_length > 21 give T4_E_INVAL, reads longer than T4_MAX_READ_LEN T4_E_UNSUPPORTED.
int T4_API( barcode_kmer_count_stats )( const char *read_pool, size_t pool_bytes, const uint64_t *seq_off, const int32_t *len,
	const int32_t *barcode, int64_t n, int kmer_length, int32_t *bc_min_cnt, int32_t *bc_median_cnt, float *bc_avg_cnt )
{
	int r = ensure_up() ;
	if ( r ) return r ;
	if ( n < 0 || !read_pool || !seq_off || !len || !barcode || kmer_length < 2 || kmer_length > 21 )
	{
		set_err( "t4_barcode_kmer_count_stats: bad argument" ) ;
		return T4_E_INVAL ;
	}
	r = check_records( "t4_barcode_kmer_count_stats", pool_bytes, seq_off, len, n ) ;
	if ( r || n == 0 )
		return r ;
	u64 inst = 0 ;
	int bmax = 0 ;
	std::vector<char> present ;
	for ( i64 i = 0 ; i < n ; ++i )
	{
		if ( barcode[i] < 0 )
		{
			set_err( "t4_barcode_kmer_count_stats: negative barcode" ) ;
			return T4_E_INVAL ;
		}
		const int j = barcode[i] >> T4_KC_BC_BITS ;
		if ( j >= (int)present.size() )
			present.resize( j + 1, 0 ) ;
		present[j] = 1 ;
		if ( barcode[i] > bmax )
			bmax = barcode[i] ;
		if ( len[i] >= kmer_length )
			inst += (u64)( len[i] - kmer_length + 1 ) ;
	}
	std::vector<int> ranges ; // only the ranges that hold reads
	for ( int j = 0 ; j < (int)present.size() ; ++j )
		if ( present[j] )
			ranges.push_back( j ) ;
	const size_t tb = T4_API( kmer_count_table_bytes )( (int64_t)inst ) ;
	DevBuf m ;
	char *dPool, *dTab ;
	u64 *dOff ;
	int32_t *dLen, *dBc, *dMin, *dMed ;
	float *dAvg ;
	m.add( dPool, pool_bytes + 16 ) ; m.add( dOff, (size_t)n * 8 ) ; m.add( dLen, (size_t)n * 4 ) ; m.add( dBc, (size_t)n * 4 ) ;
	m.add( dMin, (size_t)n * 4 ) ; m.add( dMed, (size_t)n * 4 ) ; m.add( dAvg, (size_t)n * 4 ) ; m.add( dTab, tb ) ;
	r = m.alloc() ;
	if ( !r ) r = h2d( dPool, read_pool, pool_bytes ) ;
	if ( !r ) r = h2d( dOff, seq_off, (size_t)n * 8 ) ;
	if ( !r ) r = h2d( dLen, len, (size_t)n * 4 ) ;
	if ( !r ) r = h2d( dBc, barcode, (size_t)n * 4 ) ;
	T4KcParams P ;
	kc_params( P, dTab, tb, dPool, dOff, dLen, n, kmer_length, dMin, dMed, dAvg ) ;
	if ( !r ) r = dzero( dTab, P.cap * 12 + 64 ) ;
	if ( !r ) r = bc_kc_passes( P, dBc, bmax, ranges, 0 ) ;
	u64 st[4] = { 0, 0, 0, 0 } ;
	if ( !r ) r = T4_API( kmer_count_table_stats )( dTab, tb, st ) ;
	if ( !r && st[3] )
	{
		set_err( st[3] == 1 ? "t4_barcode_kmer_count_stats: count table overflow" : "t4_barcode_kmer_count_stats: barcode out of range" ) ;
		r = T4_E_INTERNAL ;
	}
	if ( !r && bc_min_cnt ) r = d2h( bc_min_cnt, dMin, (size_t)n * 4 ) ;
	if ( !r && bc_median_cnt ) r = d2h( bc_median_cnt, dMed, (size_t)n * 4 ) ;
	if ( !r && bc_avg_cnt ) r = d2h( bc_avg_cnt, dAvg, (size_t)n * 4 ) ;
	return r ;
}

int T4_API( workload_results )( t4_workload *w, int32_t *ret_codes, int8_t *strands, int32_t *rescue_ret )
{
	int r = dsync() ;
	if ( r ) return r ;
	if ( ret_codes && ( r = d2h( ret_codes, w->ret, (size_t)w->nDescs * 4 ) ) ) return r ;
	if ( strands && ( r = d2h( strands, w->strands, (size_t)w->nDescs ) ) ) return r ;
	if ( rescue_ret && ( r = d2h( rescue_ret, w->rescue, (size_t)w->nDescs * 4 ) ) ) return r ;
	return 0 ;
}

int T4_API( shard_reads )( t4_read_desc *descs, int64_t n_descs, int n_streams, int mode, int64_t *desc_off, int64_t *order )
{
	if ( mode != T4_SHARD_RANK && mode != T4_SHARD_BARCODE && mode != T4_SHARD_GENE )
	{
		set_err( "t4_shard_reads: unknown mode" ) ;
		return T4_E_INVAL ;
	}
	int S = t4shard::Shard( descs, n_descs, n_streams, mode, desc_off, order ) ;
	if ( S < 0 )
	{
		set_err( "t4_shard_reads: bad arguments or inconsistent eq_lo / eq_hi / mate_idx" ) ;
		return T4_E_INVAL ;
	}
	return S ;
}

int T4_API( workload_events )( t4_workload *w, uint8_t *events )
{
	if ( !w || !events )
		return T4_E_INVAL ;
	int r = dsync() ;
	if ( r ) return r ;
	return d2h( events, w->events, (size_t)w->nDescs ) ;
}

int T4_API( streams_pack_contigs )( t4_seqset *const *sets, int n_sets, void *dev_buf, size_t cap, size_t *bytes_needed, int64_t *n_contigs )
{
	if ( n_sets <= 0 )
		return T4_E_INVAL ;
	std::vector<u64> so( n_sets ), sizes( n_sets ), counts( n_sets ), off( n_sets ) ;
	for ( int j = 0 ; j < n_sets ; ++j )
	{
		int r = check( sets[j] ) ;
		if ( r ) return r ;
		so[j] = sets[j]->off ;
	}
	int r = dsync() ;
	if ( r ) return r ;
	r = ensure_stage( (size_t)n_sets * 32 + 256 ) ;
	if ( r ) return r ;
	u64 *dSo = (u64 *)E.stage, *dSz = dSo + n_sets, *dCnt = dSz + n_sets, *dOff = dCnt + n_sets ;
	if ( ( r = h2d( dSo, so.data(), (size_t)n_sets * 8 ) )
		|| ( r = launch_blocks( T4_KERNEL( t4_pack_size_kernel, t4_pack_size_block ), n_sets, 128, E.A, dSo, dSz, dCnt ) )
		|| ( r = d2h( sizes.data(), dSz, (size_t)n_sets * 8 ) ) || ( r = d2h( counts.data(), dCnt, (size_t)n_sets * 8 ) ) )
		return r ;
	u64 tot = 0, n = 0 ;
	for ( int j = 0 ; j < n_sets ; ++j )
	{
		off[j] = tot ;
		tot += sizes[j] ;
		n += counts[j] ;
	}
	if ( bytes_needed ) *bytes_needed = tot ;
	if ( n_contigs ) *n_contigs = (int64_t)n ;
	if ( !dev_buf )
		return 0 ;
	if ( cap < tot )
	{
		set_err( "pack buffer too small" ) ;
		return T4_E_INVAL ;
	}
	r = h2d( dOff, off.data(), (size_t)n_sets * 8 ) ;
	if ( r ) return r ;
	return launch_blocks( T4_KERNEL( t4_pack_kernel, t4_pack_block ), n_sets, 128, E.A, dSo, dOff, (char *)dev_buf ) ;
}

// Diagnostics: SM clock cycles the last op took on each stream.
int T4_API( streams_cycles )( t4_seqset *const *sets, int n_sets, uint64_t *cycles )
{
	for ( int j = 0 ; j < n_sets ; ++j )
	{
		T4Stream st ;
		int r = get_stream( sets[j], &st ) ;
		if ( r ) return r ;
		cycles[j] = st.nReads ;
	}
	return 0 ;
}

// first device-side error among the given streams (0 if none)
int T4_API( streams_error )( t4_seqset *const *sets, int n_sets )
{
	// fast path: one word in the arena header says whether any stream raised an error since the last reset
	if ( !E.up )
		return T4_E_INVAL ;
	int r = dsync() ;
	if ( r ) return r ;
	u64 fe = 0 ;
	r = d2h( &fe, E.A + offsetof( T4Global, firstError ), sizeof( u64 ) ) ;
	if ( r ) return r ;
	if ( fe == 0 )
		return 0 ;
	for ( int j = 0 ; j < n_sets ; ++j )
	{
		T4Stream st ;
		r = get_stream( sets[j], &st ) ;
		if ( r ) return r ;
		if ( st.error )
		{
			set_err( "stream " + std::to_string( j ) + ": device error " + std::to_string( st.error ) + " aux " + std::to_string( st.errorAux ) ) ;
			return st.error ;
		}
	}
	return 0 ;
}

int T4_API( streams_run )( t4_seqset *const *sets, int n_sets, const t4_run_cfg *cfg, const t4_read_desc *descs, const int64_t *desc_off,
	const char *read_pool, size_t read_pool_bytes, const char *const *names, int n_names, int32_t *ret_codes, int8_t *strands,
	int32_t *rescue_ret )
{
	if ( n_sets <= 0 )
		return T4_E_INVAL ;
	t4_workload *w = workload_upload_impl( descs, desc_off[n_sets], read_pool, read_pool_bytes, names, n_names, true ) ;
	if ( !w )
		return T4_E_NOMEM ;
	int r = T4_API( streams_run_resident )( sets, n_sets, cfg, w, desc_off, 0 ) ;
	if ( !r )
		r = T4_API( workload_results )( w, ret_codes, strands, rescue_ret ) ;
	if ( !r )
		r = T4_API( streams_error )( sets, n_sets ) ;
	T4_API( workload_free )( w ) ;
	return r ;
}

int T4_API( seqset_add_reads_batch )( t4_seqset *s, const t4_run_cfg *cfg, const t4_read_desc *descs, int n, const char *read_pool,
	size_t read_pool_bytes, const char *const *names, int n_names, int32_t *ret_codes, int8_t *strands, int32_t *rescue_ret )
{
	int64_t off[2] = { 0, n } ;
	return T4_API( streams_run )( &s, 1, cfg, descs, off, read_pool, read_pool_bytes, names, n_names, ret_codes, strands, rescue_ret ) ;
}

} // extern "C"
