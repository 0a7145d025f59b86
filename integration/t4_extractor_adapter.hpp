// Reference-side binding of libtrust4_b200.so for stage 0: what a TRUST4 maintainer adds to run `fastq-extractor`'s
// candidate test on the GPU.  Force-included in front of the reference FastqExtractor.cpp as make_extractor_main.py
// patches it (integration/Makefile: g++ -include t4_extractor_adapter.hpp _build/extractor_main.cpp -ltrust4_b200):
//   * every -t runs the reference's batched branch (FastqExtractor.cpp:551-720), with batches of at least 2^18 reads;
//   * for each batch, before the worker threads start (:627), one t4_refset_scan call over read 1 and, with mates, one
//     over read 2 computes IsLowComplexity and HasHitInSet( read, 0 ) for every read on the device;
//   * the threads' IsGoodCandidate calls (:209, :212) get the recorded answer of their batch slot; the rest of
//     ProcessReads_Thread -- the mate rule, the barcode low-complexity rule (:215-221) -- and all of the file handling,
//     barcode correction and ReadFormatter output stay the reference's own code.
// Reads longer than T4_MAX_READ_LEN (which the scan refuses) are left out of the device batch and answered by the
// reference's own IsGoodCandidate on the host.  Any device error stops the run with t4_last_error(); there is no CPU
// fall-back.  The binary is a drop-in `fastq-extractor`: same flags, same .fq / _bc.fa / _umi.fa
// (tests/test_extractor_cli.py and tests/test_gpu_extractor.py compare them byte for byte with the stock binary).
#ifndef T4_EXTRACTOR_ADAPTER_HPP
#define T4_EXTRACTOR_ADAPTER_HPP

#ifdef T4_ADAPTER_EMU /* test build against the CPU emulation library (tests/emu): same ABI, t4emu_ prefix */
#define t4_init t4emu_init
#define t4_refset_create_from_fa t4emu_refset_create_from_fa
#define t4_refset_free t4emu_refset_free
#define t4_refset_size t4emu_refset_size
#define t4_refset_name t4emu_refset_name
#define t4_refset_set_hit_len_required t4emu_refset_set_hit_len_required
#define t4_refset_scan t4emu_refset_scan
#define t4_last_error t4emu_last_error
#endif

#include <stdint.h>
#include <time.h>
#include <string>
#include <vector>
#include "SeqSet.hpp"
#include "trust4_b200.h"

// Device arena of the run (t4_init; T4_ARENA_MB overrides it): the gene set plus one scan shell per resident worker CTA
// (about 1.2 MB each, 528 on an H100) and the hit buffers they grow.  The default of t4_init (half of the free HBM) is
// far more than stage 0 needs.
#ifdef T4_ADAPTER_EMU
#define T4_STAGE0_ARENA_BYTES ( (size_t)256 << 20 )
#else
#define T4_STAGE0_ARENA_BYTES ( (size_t)4096 << 20 )
#endif
#define T4_STAGE0_MIN_BATCH ( 1 << 18 )

static double t4_stage0_now()
{
	struct timespec t ;
	clock_gettime( CLOCK_MONOTONIC, &t ) ;
	return t.tv_sec + 1e-9 * t.tv_nsec ;
}

class T4Stage0
{
	t4_refset *ref ;
	std::vector<int8_t> answer[2] ;      // per batch slot and mate: 1 / 0 = IsGoodCandidate's result, -1 = ask the host
	std::string pool ;
	std::vector<uint64_t> off ;
	std::vector<int32_t> len ;
	std::vector<int> slot ;
	std::vector<int8_t> strand ;
	std::vector<uint8_t> low ;
	long long devReads, hostReads ;
	int batches ;
	double setSec, scanSec ;

	static void Die( const char *what )
	{
		fprintf( stderr, "trust4_b200: %s: %s\n", what, t4_last_error() ) ;
		exit( 1 ) ;
	}

	// The device gene set: the driver's -f file at refSet's k and hitLenRequired (FastqExtractor.cpp:281-282, 436-455),
	// checked against the driver's own refSet sequence by sequence.
	template <class RefSet>
	void Open( RefSet &refSet, int kmerLength, int hitLenRequired )
	{
		const double t0 = t4_stage0_now() ;
		if ( fa.size() != 1 )
		{
			fprintf( stderr, "trust4_b200: the device gene set is built from one -f file (%d given)\n", (int)fa.size() ) ;
			exit( 1 ) ;
		}
		int rc = t4_init( -1, T4_STAGE0_ARENA_BYTES ) ;
		if ( rc < 0 )
			Die( "t4_init" ) ;
		ref = t4_refset_create_from_fa( fa[0].c_str(), kmerLength ) ;
		if ( !ref )
			Die( "t4_refset_create_from_fa" ) ;
		if ( t4_refset_set_hit_len_required( ref, hitLenRequired ) < 0 )
			Die( "t4_refset_set_hit_len_required" ) ;
		const int ng = t4_refset_size( ref ) ;
		bool same = ng == refSet.Size() ;
		for ( int i = 0 ; same && i < ng ; ++i )
			same = !strcmp( t4_refset_name( ref, i ), refSet.GetSeqName( i ) ) ;
		if ( !same )
		{
			fprintf( stderr, "trust4_b200: the device gene set differs from the driver's (%d vs %d sequences)\n", ng, refSet.Size() ) ;
			exit( 1 ) ;
		}
		setSec = t4_stage0_now() - t0 ;
	}

	// One scan over the reads of one mate of the batch; reads the device refuses stay with the host.
	template <class Read>
	void ScanMate( int mate, Read *batch, int n )
	{
		pool.clear() ; off.clear() ; len.clear() ; slot.clear() ;
		answer[mate].assign( n, -1 ) ;
		for ( int i = 0 ; i < n ; ++i )
		{
			const int l = (int)strlen( batch[i].seq ) ;
			if ( l > T4_MAX_READ_LEN )
			{
				++hostReads ;
				continue ;
			}
			off.push_back( pool.size() ) ;
			len.push_back( l ) ;
			slot.push_back( i ) ;
			pool.append( batch[i].seq, l ) ;
		}
		const int64_t m = (int64_t)slot.size() ;
		if ( m == 0 )
			return ;
		pool.append( 16, '\0' ) ;
		strand.resize( m ) ;
		low.resize( m ) ;
		const double t0 = t4_stage0_now() ;
		if ( t4_refset_scan( ref, pool.data(), pool.size(), off.data(), len.data(), m, strand.data(), low.data(), NULL ) < 0 )
			Die( "t4_refset_scan" ) ;
		scanSec += t4_stage0_now() - t0 ;
		for ( int64_t j = 0 ; j < m ; ++j )
			answer[mate][ slot[j] ] = ( !low[j] && strand[j] != 0 ) ? 1 : 0 ; // IsGoodCandidate, FastqExtractor.cpp:131
		devReads += m ;
	}

public:
	std::vector<std::string> fa ; // the -f files, in the order the driver loads them (T4ExtractorRefSet::InputRefFa)

	T4Stage0() : ref( NULL ), devReads( 0 ), hostReads( 0 ), batches( 0 ), setSec( 0 ), scanSec( 0 ) {}

	static int BatchSize( int threadCnt )
	{
		if ( threadCnt < 1 )
			return 512 * threadCnt ; // what the reference does with such a -t (no reads are processed)
		return 512 * threadCnt > T4_STAGE0_MIN_BATCH ? 512 * threadCnt : T4_STAGE0_MIN_BATCH ;
	}

	// T4_EXTRACT_SCAN(): one batch, read by the reference's GetBatch calls; the worker threads start right after.
	template <class RefSet, class Read>
	void Scan( RefSet &refSet, int kmerLength, int hitLenRequired, Read *readBatch, Read *readBatch2, int batchSize, int threadCnt )
	{
		if ( ref == NULL )
			Open( refSet, kmerLength, hitLenRequired ) ;
		// At -t 1 the reference takes its per-read branch (:492-550), where ReadFiles::Next strips a trailing "/1" or "/2"
		// from the read id (ReadFiles.hpp:179-185) and that id names the read in every output file; GetBatch keeps the id
		// as it is.  Stripping it here gives the per-read branch's output.
		if ( threadCnt == 1 )
			for ( int i = 0 ; i < batchSize ; ++i )
			{
				char *id = readBatch[i].id ;
				const size_t l = strlen( id ) ;
				if ( l >= 2 && ( id[l - 1] == '1' || id[l - 1] == '2' ) && id[l - 2] == '/' )
					id[l - 2] = '\0' ;
			}
		ScanMate( 0, readBatch, batchSize ) ;
		if ( readBatch2 != NULL )
			ScanMate( 1, readBatch2, batchSize ) ;
		++batches ;
	}

	bool OnHost( int mate, int i ) const { return answer[mate][i] < 0 ; }
	int Answer( int mate, int i ) const { return answer[mate][i] ; }

	// T4_EXTRACT_DONE(), after the last batch: the gene set is released while the device is still up (not at exit).
	void Done()
	{
		if ( ref )
			t4_refset_free( ref ) ;
		ref = NULL ;
		fprintf( stderr, "[trust4_b200] stage-0 route: %lld reads scanned on the device, %lld on the host (%d batches; gene set %.3f s, "
			"device scan %.3f s)\n", devReads, hostReads, batches, setSec, scanSec ) ;
	}
} ;

static T4Stage0 t4_stage0 ;

// The driver's gene set (`SeqSet refSet( kmerLength )`, FastqExtractor.cpp:282): the reference's own object, which also
// answers the long reads on the host; the adapter only notes the -f file it loads (:318).
class T4ExtractorRefSet : public SeqSet
{
public:
	T4ExtractorRefSet( int kl ) : SeqSet( kl ) {}
	void InputRefFa( char *filename, bool isIMGT = false, const char *imgtAdditionalGap = NULL )
	{
		t4_stage0.fa.push_back( filename ) ;
		SeqSet::InputRefFa( filename, isIMGT, imgtAdditionalGap ) ;
	}
} ;

// The patched places of FastqExtractor.cpp (make_extractor_main.py).
#define T4_EXTRACT_SERIAL( threadCnt ) false
#define T4_EXTRACT_BATCH_SIZE( threadCnt ) T4Stage0::BatchSize( threadCnt )
#define T4_EXTRACT_SCAN() t4_stage0.Scan( refSet, kmerLength, hitLenRequired, readBatch, readBatch2, batchSize, threadCnt )
#define T4_EXTRACT_CANDIDATE( mate, i, read, buffer, refSet ) \
	( t4_stage0.OnHost( mate, i ) ? IsGoodCandidate( read, buffer, refSet ) : t4_stage0.Answer( mate, i ) )
#define T4_EXTRACT_DONE() t4_stage0.Done()

#define SeqSet T4ExtractorRefSet
#endif
