// Reference-side binding of libtrust4_b200.so: what a TRUST4 maintainer adds to run stage 1 (`trust4`, main.cpp)
// on the GPU without touching main.cpp.  Force-included in front of the UNMODIFIED reference main.cpp
// (integration/Makefile: g++ -include t4_seqset_adapter.hpp <reference>/main.cpp -ltrust4_b200), it
//   * derives from the reference SeqSet, so everything outside the hot path (reference gene set, rough annotation,
//     AssignRead / mate extension, RemoveRedundantSeq) keeps running the reference's own CPU code;
//   * routes the novel-contig set of the stage-1 driver (`SeqSet seqSet`, main.cpp:642 -- the first SeqSet constructed)
//     through the C ABI of include/trust4_b200.h: AddRead, RepeatAddRead, InputNovelRead, UpdateAllConsensus,
//     ChangeKmerLength, Size, SetHitLenRequired, Output (SeqSet.hpp:3426, 4477, 3028, 4525, 4624, 2591, 2601, 10939),
//     ReleaseFinishedBarcodeSeq, ReleaseShallowContigs, InputNovelFa (SeqSet.hpp:10815, 10928, 2986);
//   * hands the contigs back to the CPU object after the assembly (Output is the driver's first use of them,
//     main.cpp:1957-1975) so that `extendedSeq.InputSeqSet( seqSet, false )` (main.cpp:2049) sees them.
// The resulting binary is a drop-in `trust4`: same flags, same _raw.out / _final.out / _assembled_reads.fa
// (tests/test_dropin_cli.py compares them byte for byte with the stock binary).
#ifndef T4_SEQSET_ADAPTER_HPP
#define T4_SEQSET_ADAPTER_HPP

#ifdef T4_ADAPTER_EMU /* test build against the CPU emulation library (tests/emu): same ABI, t4emu_ prefix */
#define t4_seqset_create t4emu_seqset_create
#define t4_seqset_destroy t4emu_seqset_destroy
#define t4_seqset_add_read t4emu_seqset_add_read
#define t4_seqset_repeat_add_read t4emu_seqset_repeat_add_read
#define t4_seqset_input_novel_read t4emu_seqset_input_novel_read
#define t4_seqset_update_all_consensus t4emu_seqset_update_all_consensus
#define t4_seqset_change_kmer_length t4emu_seqset_change_kmer_length
#define t4_seqset_size t4emu_seqset_size
#define t4_seqset_kmer_length t4emu_seqset_kmer_length
#define t4_seqset_set_hit_len_required t4emu_seqset_set_hit_len_required
#define t4_seqset_set_is_long t4emu_seqset_set_is_long
#define t4_seqset_set_consider_barcode_in_hash t4emu_seqset_set_consider_barcode_in_hash
#define t4_seqset_output t4emu_seqset_output
#define t4_seqset_get_contig t4emu_seqset_get_contig
#define t4_seqset_contig_flags t4emu_seqset_contig_flags
#define t4_seqset_release_finished_barcode t4emu_seqset_release_finished_barcode
#define t4_seqset_release_shallow_contigs t4emu_seqset_release_shallow_contigs
#define t4_seqset_input_novel_fa t4emu_seqset_input_novel_fa
#define t4_seqsets_create_ex t4emu_seqsets_create_ex
#define t4_workload_upload t4emu_workload_upload
#define t4_workload_free t4emu_workload_free
#define t4_streams_run_resident t4emu_streams_run_resident
#define t4_workload_results t4emu_workload_results
#define t4_workload_events t4emu_workload_events
#define t4_shard_reads t4emu_shard_reads
#define t4_streams_error t4emu_streams_error
#define t4_streams_assign_reads t4emu_streams_assign_reads
#define t4_assign_results t4emu_assign_results
#define t4_assign_extended_set t4emu_assign_extended_set
#define t4_assign_free t4emu_assign_free
#define t4_refset_create_from_fa t4emu_refset_create_from_fa
#define t4_refset_free t4emu_refset_free
#define t4_refset_size t4emu_refset_size
#define t4_refset_name t4emu_refset_name
#define t4_refset_set_hit_len_required t4emu_refset_set_hit_len_required
#define t4_refset_set_radius t4emu_refset_set_radius
#define t4_refset_annotate t4emu_refset_annotate
#define t4_kmer_count_stats t4emu_kmer_count_stats
#define t4_sort_reads t4emu_sort_reads
#define t4_barcode_kmer_count_stats t4emu_barcode_kmer_count_stats
#define t4_sort_reads_barcode t4emu_sort_reads_barcode
#define t4_last_error t4emu_last_error
#define t4_init t4emu_init
#endif

#include <stdarg.h>
#include <time.h>
#include <assert.h>
#include <limits.h>
#include <map>
#include <string>
#include <vector>
#define private public /* the adapter refills SeqSet::seqs from the device */
#include "SeqSet.hpp"
#undef private
#include "trust4_b200.h"

static int t4_adapter_instances = 0 ;
static std::string t4_adapter_ref_fa ; // the -f file, noted when the driver loads its reference gene set (main.cpp:674)

class T4GpuSeqSet : public SeqSet
{
	t4_seqset *h ;
	bool gpu ;
	// ---- batch route (T4_BATCH_PREPARE, below): the device runs the whole loop, the driver's own loop replays it ----
	std::vector<t4_seqset *> sets ;      // sets[0] == h
	bool replay ;
	int curK, curHitLen, curConsiderBarcode ;
	std::vector<int32_t> bRet, bResc ;
	std::vector<int8_t> bStrand ;
	std::vector<uint8_t> bEv ;
	std::vector<int> rescueOrder ;
	size_t cur, rescuePos ;
	int maxFinalK ;
	t4_workload *wl ;                    // the uploaded read list, kept for the AssignRead pass (BatchAssign)
	std::vector<int64_t> wlOff, wlOrder ;
	void Die() { fprintf( stderr, "trust4_b200: %s\n", t4_last_error() ) ; exit( 1 ) ; }
	int Check( int r ) { if ( r < T4_E_BASE ) Die() ; return r ; }

	// Copy the device contigs into the CPU object (slot numbers preserved; released slots stay NULL).
	void SyncToHost()
	{
		for ( size_t i = 0 ; i < seqs.size() ; ++i )
		{
			if ( seqs[i].consensus ) free( seqs[i].consensus ) ;
			if ( seqs[i].name ) free( seqs[i].name ) ;
		}
		seqs.clear() ;
		std::vector<char> cons, name( 4096 ) ;
		std::vector<int32_t> pw ;
		std::map<int, int> purgedBarcodes ;
		// read-sharded batch runs hold one device set per stream: the mirror is their concatenation in stream order
		// (global slot = local slot + slots of the earlier streams, SURVEY.md 8e)
		for ( size_t si = 0 ; si < sets.size() ; ++si )
		{
		t4_seqset *h = sets[si] ;
		int n = Check( t4_seqset_size( h ) ) ;
		for ( int i = 0 ; i < n ; ++i )
		{
			struct _seqWrapper ns ;
			ns.name = ns.consensus = NULL ;
			ns.consensusLen = 0 ;
			ns.isRef = false ;
			ns.minLeftExtAnchor = ns.minRightExtAnchor = 0 ;
			ns.barcode = -1 ;
			ns.numRead = 0 ;
			ns.index = true ;
			ns.posWeightCompressed = false ;
			for ( int j = 0 ; j < 3 ; ++j )
				ns.info[j].a = ns.info[j].b = ns.info[j].c = 0 ;
			int len = t4_seqset_get_contig( h, i, NULL, 0, NULL, NULL, 0, NULL, NULL, NULL, NULL ) ;
			if ( len >= 0 )
			{
				cons.resize( len + 1 ) ;
				pw.resize( 4 * (size_t)len + 4 ) ;
				Check( t4_seqset_get_contig( h, i, cons.data(), len + 1, pw.data(), name.data(), (int)name.size(), &ns.barcode,
					&ns.numRead, &ns.minLeftExtAnchor, &ns.minRightExtAnchor ) ) ;
				ns.consensus = strdup( cons.data() ) ;
				ns.name = strdup( name.data() ) ;
				ns.consensusLen = len ;
				if ( Check( t4_seqset_contig_flags( h, i ) ) & T4_CONTIG_PURGED )
					purgedBarcodes[ns.barcode] = 1 ;
			}
			seqs.push_back( ns ) ;
			if ( len >= 0 )
			{
				struct _seqWrapper &sw = seqs.back() ;
				sw.posWeight.ExpandTo( len ) ;
				for ( int j = 0 ; j < len ; ++j )
					for ( int k = 0 ; k < 4 ; ++k )
						sw.posWeight[j].count[k] = pw[4 * j + k] ;
			}
		}
		}
		// Contigs the device purged (ReleaseFinishedBarcodeSeq) keep their full posWeight columns there; the reference
		// compresses or frees them and marks them un-indexed.  Re-apply exactly that storage change to the mirror with the
		// reference's own code (the index removal and UpdateConsensus inside it are no-ops here: the host index is empty
		// and the consensus is already final), so everything downstream of Output sees the reference's object state.
		if ( !purgedBarcodes.empty() )
			SeqSet::ReleaseFinishedBarcodeSeq( purgedBarcodes, true, 0, false ) ;
	}
public:
	T4GpuSeqSet( int kl ) : SeqSet( kl ), h( NULL ), replay( false ), curK( kl ), curHitLen( 31 ), curConsiderBarcode( 0 ), cur( 0 ), rescuePos( 0 ),
		maxFinalK( kl ), wl( NULL )
	{
		gpu = ( t4_adapter_instances++ == 0 ) ;
		if ( gpu )
		{
			h = t4_seqset_create( kl ) ;
			if ( !h )
				Die() ;
			sets.push_back( h ) ;
		}
	}
	~T4GpuSeqSet()
	{
		if ( wl )
			t4_workload_free( wl ) ;
		for ( size_t i = 0 ; i < sets.size() ; ++i )
			t4_seqset_destroy( sets[i] ) ;
	}

	// ---- the batch route ---------------------------------------------------------------------------------------------
	// T4_BATCH_PREPARE() is the ONE line added to main.cpp, directly in front of the AddRead loop (main.cpp:1583).  When the
	// environment variable T4_STREAMS = S >= 1 is set, it restates the loop's per-read preparation (main.cpp:1596-1745: the
	// duplicate test, the V/D/J/C order and constant-gene filters, gene prefix / strand / similarity threshold /
	// minKmerCount of the AddRead call, the may-seed-a-contig rule, the mate hints) into t4_read_desc records, runs the
	// whole loop and the rescue pass on the device (S = 1: one stream = the reference's serial semantics; S > 1: S
	// contiguous shards of the sorted list, one SeqSet each) and arms `replay`: the driver's own unmodified loop then
	// asks AddRead / RepeatAddRead / InputNovelRead / Size again and gets the device's answers, so all of its
	// bookkeeping (assembledReadIdx, strands, rescue list, k) ends up exactly as if it had done the work.
	template <class Reads, class RefSet>
	void BatchPrepare( Reads &sortedReads, RefSet &refSet, int readCnt, bool hasBarcode, bool keepMissingBarcode, int trimLevel,
		int firstReadLen, int constantGeneEnd, int contigMinCov, int changeKmerLengthThreshold )
	{
		const char *env = getenv( "T4_STREAMS" ) ;
		if ( !gpu || env == NULL || atoi( env ) < 1 || readCnt <= 0 )
			return ;
		int S = atoi( env ) ;
		const int n = readCnt ;
		std::vector<t4_read_desc> d( n ) ;
		std::string pool ;
		std::vector<std::string> names ;
		std::map<std::string, int> nameId ;
		struct _overlap go[4] ;
		memset( go, 0, sizeof( go ) ) ;
		for ( int j = 0 ; j < 4 ; ++j )
			go[j].seqIdx = -1 ;
		int runLo = 0 ;
		uint32_t runGood = 0 ;
		for ( int i = 0 ; i < n ; ++i )
		{
			t4_read_desc &r = d[i] ;
			memset( &r, 0, sizeof( r ) ) ;
			const char *read = sortedReads[i].read ;
			const int len = (int)strlen( read ) ;
			if ( len > T4_MAX_READ_LEN )
			{
				fprintf( stderr, "trust4_b200: read longer than %d bases\n", T4_MAX_READ_LEN ) ;
				exit( 1 ) ;
			}
			const bool sameString = i > 0 && !strcmp( read, sortedReads[i - 1].read ) ;
			const bool dup = sameString && sortedReads[i].barcode == sortedReads[i - 1].barcode ; // main.cpp:1596
			if ( !sameString )
				runLo = i ;
			r.seq_off = pool.size() ;
			pool.append( read, len ) ;
			r.len = len ;
			r.barcode = sortedReads[i].barcode ;
			r.min_cnt = sortedReads[i].minCnt ;
			r.min_kmer_count = hasBarcode ? ( sortedReads[i].minCnt + sortedReads[i].barcodeMinCnt + 1 ) / 2 : sortedReads[i].minCnt ;
			r.sim_threshold = 0.9 ;
			r.name_id = -1 ;
			r.mate_idx = sortedReads[i].mateIdx ;
			r.eq_lo = runLo ;
			if ( dup )
			{
				r.flags = T4_RD_DUP | runGood ; // the static geneOverlap of main.cpp:1588 still holds the run's first read
				continue ;
			}
			for ( int j = 0 ; j < 4 ; ++j )
				go[j] = sortedReads[i].geneOverlap[j] ;
			bool filter = false ;
			for ( int j = 0 ; j < 4 && !filter ; ++j ) // main.cpp:1620-1638
			{
				if ( go[j].seqIdx == -1 )
					continue ;
				for ( int l = j + 1 ; l < 4 ; ++l )
					if ( go[l].seqIdx != -1 && go[j].readEnd - 10 > go[l].readStart )
					{
						filter = true ;
						break ;
					}
			}
			if ( go[3].seqIdx != -1 && go[0].seqIdx == -1 && go[2].seqIdx == -1 ) // main.cpp:1640-1651
			{
				if ( go[3].seqStart >= constantGeneEnd )
					filter = true ;
				else if ( constantGeneEnd <= 200 && go[3].seqStart >= 100
					&& ( go[3].strand == 1 || go[3].readEnd - go[3].readStart + 1 < sortedReads[i].len ) )
					filter = true ;
			}
			uint32_t fl = 0 ;
			if ( filter )
				fl |= T4_RD_FILTERED ;
			else
			{
				char name[5] = "" ;
				int strand = 0, ambiguous = 0 ;
				for ( int j = 0 ; j < 4 ; ++j ) // main.cpp:1660-1673
					if ( go[j].seqIdx != -1 )
					{
						char *sn = refSet.GetSeqName( go[j].seqIdx ) ;
						name[0] = sn[0] ; name[1] = sn[1] ; name[2] = sn[2] ; name[3] = sn[3] ; name[4] = '\0' ;
						if ( strand != 0 && strand != go[j].strand )
							ambiguous = 1 ;
						strand = go[j].strand ;
					}
				if ( ambiguous )
					strand = 0 ;
				double thr = 0.9 ; // main.cpp:1675-1694
				if ( sortedReads[i].minCnt >= 20 )
					thr = 0.97 ;
				else if ( sortedReads[i].minCnt >= 2 || ( sortedReads[i].minCnt >= 5 && firstReadLen > 200 ) )
					thr = 0.95 ;
				if ( name[0] == 'T' && thr < 0.95 )
					thr = 0.95 ;
				if ( hasBarcode || trimLevel > 1 )
					thr = 0.9 ;
				r.sim_threshold = thr ;
				r.strand_in = (int8_t)strand ;
				for ( int j = 0 ; j < 4 ; ++j )
					r.gene4[j] = name[j] ;
				// main.cpp:1704-1745: may InputNovelRead seed a contig when AddRead fails?
				int matchCnt = 0, first = 4 ;
				for ( int j = 3 ; j >= 0 ; --j )
					if ( go[j].seqIdx != -1 )
					{
						matchCnt += go[j].matchCnt / 2 ;
						first = j ;
					}
				bool f2 = true ;
				if ( matchCnt >= 31 )
					f2 = false ;
				else if ( go[0].seqIdx != -1 && go[2].seqIdx != -1 && go[0].readEnd < go[2].readStart )
					f2 = false ;
				else if ( go[0].seqIdx != -1 )
				{
					if ( go[0].seqEnd >= refSet.GetSeqConsensusLen( go[0].seqIdx ) - 17 )
						f2 = false ;
				}
				else if ( go[2].seqIdx != -1 )
				{
					if ( go[2].seqStart <= 17 )
						f2 = false ;
				}
				if ( !f2 && first < 4 )
				{
					fl |= T4_RD_NOVEL_ON_FAIL ;
					std::string gn( refSet.GetSeqName( go[first].seqIdx ) ) ;
					std::map<std::string, int>::iterator it = nameId.find( gn ) ;
					if ( it == nameId.end() )
					{
						nameId[gn] = (int)names.size() ;
						r.name_id = (int)names.size() ;
						names.push_back( gn ) ;
					}
					else
						r.name_id = it->second ;
					r.novel_strand = (int8_t)go[first].strand ;
				}
				if ( SeqSet::HasMotif( sortedReads[i].read, 1 ) ) // main.cpp:1752 (the result does not depend on the sign)
					fl |= T4_RD_MOTIF ;
			}
			// main.cpp:1782-1808 for either outcome of sortedReads[i].strand; consulted only when the read was added
			runGood = 0 ;
			for ( int sgn = 1 ; sgn >= -1 ; sgn -= 2 )
			{
				bool good = false, maySpan = false ;
				if ( go[0].seqIdx != -1 && go[0].similarity >= 0.9 && sgn == 1 )
				{
					good = true ;
					if ( go[2].seqIdx != -1 && go[2].readStart > go[0].readEnd ) maySpan = true ;
					if ( go[3].seqIdx != -1 && go[3].readStart > go[0].readEnd ) maySpan = true ;
				}
				for ( int j = 2 ; j <= 3 ; ++j )
					if ( go[j].seqIdx != -1 && go[j].similarity >= 0.9 && sgn == -1 )
					{
						good = true ;
						if ( go[0].seqIdx != -1 && go[j].readStart > go[0].readEnd ) maySpan = true ;
					}
				if ( maySpan )
					good = false ;
				if ( good )
					runGood |= ( sgn == 1 ) ? T4_RD_GOOD_PLUS : T4_RD_GOOD_MINUS ;
			}
			r.flags = fl | runGood ;
		}
		for ( int i = n - 1, hi = n ; i >= 0 ; --i ) // eq_hi: end of the run of identical read strings (main.cpp:1826-1835)
		{
			d[i].eq_hi = hi ;
			if ( d[i].eq_lo == i )
				hi = i ;
		}
		// streams (SURVEY.md 8e): T4_SHARD_BY = gene (default without barcodes: reads grouped by annotated gene, so a
		// clonotype's reads meet in one SeqSet) | rank (contiguous blocks of the sorted list); whole barcodes with --barcode.
		// Neither splits a run of identical reads; S = 1 is the identity.
		const char *by = getenv( "T4_SHARD_BY" ) ;
		int mode = hasBarcode ? T4_SHARD_BARCODE : ( by && !strcmp( by, "rank" ) ) ? T4_SHARD_RANK : T4_SHARD_GENE ;
		std::vector<int64_t> off( ( S > n ? n : S ) + 1, 0 ), order( n ) ;
		S = t4_shard_reads( d.data(), n, S, mode, off.data(), order.data() ) ;
		if ( S < 1 )
			Die() ;
		off.resize( S + 1 ) ;
		if ( S > 1 )
		{
			sets.resize( S ) ;
			Check( t4_seqsets_create_ex( S - 1, curK, curHitLen, curConsiderBarcode, sets.data() + 1 ) ) ;
		}
		t4_run_cfg cfg ;
		memset( &cfg, 0, sizeof( cfg ) ) ;
		cfg.has_barcode = hasBarcode ;
		cfg.repetitive = trimLevel > 1 ;
		cfg.change_k_threshold = changeKmerLengthThreshold ;
		cfg.update_consensus_every = 10000 ;
		cfg.do_rescue = 1 ;
		cfg.first_read_len = firstReadLen ;
		cfg.final_update = 1 ;
		cfg.release_barcodes = hasBarcode && !keepMissingBarcode ;
		cfg.contig_min_cov = contigMinCov ;
		std::vector<const char *> np ;
		for ( size_t i = 0 ; i < names.size() ; ++i )
			np.push_back( names[i].c_str() ) ;
		pool.append( 16, '\0' ) ;
		t4_workload *w = t4_workload_upload( d.data(), n, pool.data(), pool.size(), np.data(), (int)np.size() ) ;
		if ( !w )
			Die() ;
		Check( t4_streams_run_resident( sets.data(), S, &cfg, w, off.data(), NULL ) ) ;
		bRet.resize( n ) ; bResc.resize( n ) ; bStrand.resize( n ) ; bEv.resize( n ) ;
		{
			std::vector<int> ret( n ), resc( n ) ;
			std::vector<int8_t> str( n ) ;
			std::vector<uint8_t> ev( n ) ;
			Check( t4_workload_results( w, ret.data(), str.data(), resc.data() ) ) ;
			Check( t4_workload_events( w, ev.data() ) ) ;
			for ( int j = 0 ; j < n ; ++j ) // back to the driver's order: the replay walks sortedReads
			{
				const int64_t i = order[j] ;
				bRet[i] = ret[j] ; bResc[i] = resc[j] ; bStrand[i] = str[j] ; bEv[i] = ev[j] ;
			}
		}
		Check( t4_streams_error( sets.data(), S ) ) ;
		wl = w ; // the AssignRead pass (BatchAssign) reads the same records and the per-read results on the device
		wlOff = off ;
		wlOrder = order ;
		rescueOrder.clear() ;
		for ( int i = 0 ; i < n ; ++i )
			if ( bRet[i] == -2 )
				rescueOrder.push_back( i ) ;
		int nk = 0 ;
		for ( int i = 0 ; i < n ; ++i )
			if ( bEv[i] & T4_EV_CHANGE_K )
				++nk ;
		maxFinalK = curK + 2 * ( S == 1 ? nk : ( nk > 0 ? 1 : 0 ) ) ;
		for ( int s = 0 ; S > 1 && s < S ; ++s )
		{
			int ks = Check( t4_seqset_kmer_length( sets[s] ) ) ;
			if ( ks > maxFinalK )
				maxFinalK = ks ;
		}
		replay = true ;
		cur = 0 ;
		rescuePos = 0 ;
		fprintf( stderr, "[trust4_b200] batch route: %d reads on %d device stream(s)\n", n, S ) ;
	}

	// T4_BATCH_ASSIGN() is the second inserted line of the batch route: `if ( !seqSet.BatchAssign( ... ) )` in front of the
	// driver's AssignRead loop (main.cpp:2075: `if ( threadCnt <= 1 ) { ... } else { ... pthreads ... }`), which thereby
	// becomes the fall-back branch.  The device runs the pass (t4_streams_assign_reads: extended sets by InputSeqSet at
	// extendedSeq's k, AssignRead of every assembled read with novelSeqSimilarity 0.95, worker CTAs over the whole GPU) on the
	// sets and the read list of BatchPrepare, and assembledReads[].overlap receives what the driver's own loop would have
	// stored -- including the reference's reuse of one `assign` variable: a read AssignRead cannot place only gets
	// seqIdx = -1, the other fields keep the previous assignment (main.cpp:2051, 2078-2081).  extendedSeq itself is the CPU
	// object the driver built (InputSeqSet of the synced contigs): its slots are the concatenation of the streams' extended
	// sets, so a device slot becomes a global one by adding the sizes of the earlier streams' sets.  RecomputePosWeight
	// (main.cpp:2118) then runs on the CPU object from these assignments.  T4_ASSIGN=0 keeps the pass on the CPU.
	template <class ExtSet, class AReads>
	bool BatchAssign( ExtSet &extendedSeq, AReads &assembledReads, int assembledReadCnt )
	{
		const char *env = getenv( "T4_ASSIGN" ) ;
		if ( !gpu || !replay || wl == NULL || ( env && atoi( env ) == 0 ) )
			return false ;
		const int S = (int)sets.size() ;
		const int64_t n = (int64_t)wlOrder.size() ;
		t4_assign *a = t4_streams_assign_reads( sets.data(), S, wl, wlOff.data(), extendedSeq.kmerLength, 0, NULL ) ;
		if ( !a )
			Die() ;
		std::vector<int32_t> as( 8 * (size_t)n + 8 ) ;
		std::vector<double> sim( (size_t)n + 1 ) ;
		Check( t4_assign_results( a, as.data(), sim.data() ) ) ;
		std::vector<int> base( S + 1, 0 ), streamOf( (size_t)n ) ;
		for ( int s = 0 ; s < S ; ++s )
		{
			base[s + 1] = base[s] + Check( t4_seqset_size( t4_assign_extended_set( a, s ) ) ) ;
			for ( int64_t j = wlOff[s] ; j < wlOff[s + 1] ; ++j )
				streamOf[j] = s ;
		}
		if ( base[S] != (int)extendedSeq.seqs.size() )
		{
			fprintf( stderr, "trust4_b200: extended sets out of step (%d device slots, %d host slots)\n", base[S], (int)extendedSeq.seqs.size() ) ;
			exit( 1 ) ;
		}
		std::vector<int64_t> recOf( (size_t)n ) ;
		for ( int64_t j = 0 ; j < n ; ++j )
			recOf[ wlOrder[j] ] = j ;
		struct _overlap assign ;
		memset( &assign, 0, sizeof( assign ) ) ;
		assign.seqIdx = -1 ;
		int placed = 0 ;
		for ( int x = 0 ; x < assembledReadCnt ; ++x )
		{
			const int64_t j = recOf[ assembledReads[x].info ] ;
			const int32_t *o = &as[8 * j] ;
			if ( o[0] == T4_ASSIGN_NOT_LISTED )
			{
				fprintf( stderr, "trust4_b200: assembled read %d is not part of the device's AssignRead pass\n", x ) ;
				exit( 1 ) ;
			}
			if ( o[0] >= 0 )
			{
				assign.seqIdx = o[0] + base[ streamOf[j] ] ;
				assign.readStart = o[1] ; assign.readEnd = o[2] ;
				assign.seqStart = o[3] ; assign.seqEnd = o[4] ;
				assign.strand = o[5] ;
				assign.matchCnt = o[6] ;
				assign.similarity = sim[j] ;
				++placed ;
			}
			else
				assign.seqIdx = -1 ;
			assembledReads[x].overlap = assign ;
		}
		t4_assign_free( a ) ;
		t4_workload_free( wl ) ;
		wl = NULL ;
		fprintf( stderr, "[trust4_b200] batch route: AssignRead pass on the device, %d of %d reads placed\n", placed, assembledReadCnt ) ;
		return true ;
	}

	// T4_BATCH_KMERSTATS() is the (opt-in, T4_KMERSTATS=1) line in front of the count-statistics loop (main.cpp:981:
	// `if (threadCnt == 1) { ... GetCountStatsAndTrim ... } else { pthreads }`).  The driver has filled `kmerCount` with the
	// 21-mers of every read it kept while loading (ProcessRead, main.cpp:401-440); the device counts the same reads again in
	// one HBM table and returns minCnt / medianCnt / avgCnt and the quality trim per read (t4_kmer_count_stats), and the reads
	// are cut / dropped exactly as the loop would have (main.cpp:985-1010).  Not applicable -- the CPU loop runs -- when the
	// counts came from a file (-k) or reads were removed after counting (--contigMinCov with barcodes, main.cpp:951-978).
	template <class Reads>
	bool BatchKmerStats( Reads &sortedReads, int readCnt, int trimLevel, bool countMyself, bool readsRemovedAfterCounting )
	{
		const char *env = getenv( "T4_KMERSTATS" ) ;
		if ( !gpu || env == NULL || atoi( env ) != 1 || getenv( "T4_STREAMS" ) == NULL || readCnt <= 0 || !countMyself || readsRemovedAfterCounting )
			return false ;
		std::string pool, qpool ;
		std::vector<uint64_t> off( readCnt ) ;
		std::vector<int32_t> len( readCnt ) ;
		const bool useQual = trimLevel != 0 ;
		bool allQual = true ;
		for ( int i = 0 ; i < readCnt ; ++i )
		{
			off[i] = pool.size() ;
			len[i] = (int)strlen( sortedReads[i].read ) ;
			if ( len[i] > T4_MAX_READ_LEN )
				return false ; // the CPU loop handles it (the assembly route will refuse such reads later)
			pool.append( sortedReads[i].read, len[i] ) ;
			if ( useQual )
			{
				if ( sortedReads[i].qual == NULL )
					allQual = false ;
				else
					qpool.append( sortedReads[i].qual, len[i] ) ;
			}
		}
		if ( useQual && !allQual )
			return false ; // FASTA input mixed in: per-read qual == NULL cases stay on the CPU
		pool.append( 16, '\0' ) ;
		if ( useQual )
			qpool.append( 16, '\0' ) ;
		std::vector<int32_t> mn( readCnt ), med( readCnt ), nl( readCnt ) ;
		std::vector<float> avg( readCnt ) ;
		Check( t4_kmer_count_stats( pool.data(), useQual ? qpool.data() : NULL, pool.size(), off.data(), len.data(), readCnt, 21, mn.data(),
			med.data(), avg.data(), nl.data() ) ) ;
		int trimmed = 0 ;
		for ( int i = 0 ; i < readCnt ; ++i )
		{
			sortedReads[i].minCnt = mn[i] ;
			sortedReads[i].medianCnt = med[i] ;
			sortedReads[i].avgCnt = avg[i] ;
			if ( nl[i] < len[i] )
			{
				sortedReads[i].read[ nl[i] ] = '\0' ;
				++trimmed ;
			}
			if ( sortedReads[i].qual != NULL ) // main.cpp:991-1000
			{
				free( sortedReads[i].qual ) ;
				sortedReads[i].qual = NULL ;
			}
			if ( sortedReads[i].read[0] == '\0' ) // main.cpp:1004-1009
			{
				free( sortedReads[i].read ) ;
				free( sortedReads[i].id ) ;
				sortedReads[i].read = NULL ;
			}
		}
		fprintf( stderr, "[trust4_b200] batch route: 21-mer statistics on the device, %d of %d reads trimmed\n", trimmed, readCnt ) ;
		return true ;
	}

	// T4_BATCH_SORT() (opt-in, T4_SORT=1) in front of `std::sort( sortedReads.begin(), sortedReads.end() ) ;` (main.cpp:1078),
	// which becomes the fall-back statement: the device returns the permutation of _sortRead::operator< (t4_sort_reads) and
	// the records are moved accordingly.  Emulation-verified only so far.
	template <class Reads>
	bool BatchSort( Reads &sortedReads )
	{
		const char *env = getenv( "T4_SORT" ) ;
		const int64_t n = (int64_t)sortedReads.size() ;
		if ( !gpu || env == NULL || atoi( env ) != 1 || getenv( "T4_STREAMS" ) == NULL || n <= 1 )
			return false ;
		std::string pool, idPool ;
		std::vector<uint64_t> off( n ), idOff( n + 1 ) ;
		std::vector<int32_t> len( n ), mn( n ), med( n ) ;
		std::vector<float> avg( n ) ;
		for ( int64_t i = 0 ; i < n ; ++i )
		{
			off[i] = pool.size() ;
			len[i] = (int32_t)strlen( sortedReads[i].read ) ;
			pool.append( sortedReads[i].read, len[i] ) ;
			idOff[i] = idPool.size() ;
			idPool.append( sortedReads[i].id ) ;
			mn[i] = sortedReads[i].minCnt ; med[i] = sortedReads[i].medianCnt ; avg[i] = sortedReads[i].avgCnt ;
		}
		idOff[n] = idPool.size() ;
		pool.append( 16, '\0' ) ;
		idPool.append( 16, '\0' ) ;
		std::vector<int64_t> order( n ) ;
		Check( t4_sort_reads( pool.data(), pool.size(), off.data(), len.data(), idPool.data(), idPool.size(), idOff.data(), mn.data(), med.data(),
			avg.data(), n, order.data() ) ) ;
		Reads sorted ;
		sorted.reserve( n ) ;
		for ( int64_t j = 0 ; j < n ; ++j )
			sorted.push_back( sortedReads[ order[j] ] ) ;
		sortedReads.swap( sorted ) ;
		fprintf( stderr, "[trust4_b200] batch route: %lld reads sorted on the device\n", (long long)n ) ;
		return true ;
	}

	// T4_BATCH_BARCODE_STATS() (opt-in, T4_BCSTATS=1) in front of `if (hasBarcode) { ... }` (main.cpp:1123-1194), which
	// becomes the fall-back branch.  That block sorts the reads with CompReadWithBarcode (:1126), counts 21-mers per barcode
	// group into barcodeMinCnt / barcodeMedianCnt / barcodeAvgCnt (:1128-1180), then re-sorts every barcode group with the
	// same comparator (:1183-1192).  The first sort runs while every barcodeMinCnt is still 0 (the _sortRead constructor), so
	// it only groups the reads by barcode, with operator< inside a group; the re-sort then orders each group by
	// (barcodeMinCnt desc, operator<).  Together that is ONE sort of the whole list under CompReadWithBarcode with the final
	// barcodeMinCnt, and the counting does not depend on the read order -- so the device counts first
	// (t4_barcode_kmer_count_stats, reads in the driver's current order) and sorts once (t4_sort_reads_barcode).  With
	// --barcode every read has a barcode >= 0 (main.cpp:797-819); the comparator is an order only then.  Not applicable --
	// the CPU block runs -- without --barcode, with a negative barcode, or with a read over the device's length limit.
	template <class Reads>
	bool BatchBarcodeStats( Reads &sortedReads, int readCnt, bool hasBarcode )
	{
		const char *env = getenv( "T4_BCSTATS" ) ;
		const int64_t n = readCnt ;
		if ( !gpu || env == NULL || atoi( env ) != 1 || getenv( "T4_STREAMS" ) == NULL || !hasBarcode || n <= 0 || n != (int64_t)sortedReads.size() )
			return false ;
		std::string pool, idPool ;
		std::vector<uint64_t> off( n ), idOff( n + 1 ) ;
		std::vector<int32_t> len( n ), mn( n ), med( n ), bc( n ) ;
		std::vector<float> avg( n ) ;
		for ( int64_t i = 0 ; i < n ; ++i )
		{
			off[i] = pool.size() ;
			len[i] = (int32_t)strlen( sortedReads[i].read ) ;
			if ( len[i] > T4_MAX_READ_LEN || sortedReads[i].barcode < 0 )
				return false ;
			pool.append( sortedReads[i].read, len[i] ) ;
			idOff[i] = idPool.size() ;
			idPool.append( sortedReads[i].id ) ;
			mn[i] = sortedReads[i].minCnt ; med[i] = sortedReads[i].medianCnt ; avg[i] = sortedReads[i].avgCnt ;
			bc[i] = sortedReads[i].barcode ;
		}
		idOff[n] = idPool.size() ;
		pool.append( 16, '\0' ) ;
		idPool.append( 16, '\0' ) ;
		std::vector<int32_t> bmn( n ), bmed( n ) ;
		std::vector<float> bavg( n ) ;
		Check( t4_barcode_kmer_count_stats( pool.data(), pool.size(), off.data(), len.data(), bc.data(), n, 21, bmn.data(), bmed.data(),
			bavg.data() ) ) ;
		for ( int64_t i = 0 ; i < n ; ++i )
		{
			sortedReads[i].barcodeMinCnt = bmn[i] ;
			sortedReads[i].barcodeMedianCnt = bmed[i] ;
			sortedReads[i].barcodeAvgCnt = bavg[i] ;
		}
		std::vector<int64_t> order( n ) ;
		Check( t4_sort_reads_barcode( pool.data(), pool.size(), off.data(), len.data(), idPool.data(), idPool.size(), idOff.data(), mn.data(),
			med.data(), avg.data(), bc.data(), bmn.data(), n, order.data() ) ) ;
		Reads sorted ;
		sorted.reserve( n ) ;
		for ( int64_t j = 0 ; j < n ; ++j )
			sorted.push_back( sortedReads[ order[j] ] ) ;
		sortedReads.swap( sorted ) ;
		int cells = 0 ;
		for ( int64_t j = 0 ; j < n ; ++j )
			if ( j == 0 || sortedReads[j].barcode != sortedReads[j - 1].barcode )
				++cells ;
		fprintf( stderr, "[trust4_b200] batch route: per-cell 21-mer statistics and barcode sort on the device, %lld reads in %d cells\n",
			(long long)n, cells ) ;
		return true ;
	}

	// main.cpp:674 `refSet.InputRefFa( optarg )`: the CPU object loads the genes as always; the file name is kept so that the
	// batch route can build the same gene set on the device (BatchAnnotate).
	void InputRefFa( char *filename, bool isIMGT = false, const char *imgtAdditionalGap = NULL )
	{
		if ( !gpu )
			t4_adapter_ref_fa = filename ;
		SeqSet::InputRefFa( filename, isIMGT, imgtAdditionalGap ) ;
	}

	// T4_BATCH_ANNOTATE() is the third inserted line of the batch route: `if ( !seqSet.BatchAnnotate( ... ) )` in front of the
	// rough annotation loop (main.cpp:1084: `if ( threadCnt <= 1 ) { ... AnnotateRead( read, 0, ... ) ... } else { pthreads }`),
	// which becomes the fall-back branch.  OPT-IN (T4_ANNOTATE=1): the device pass behind it (t4_refset_annotate) has been
	// verified through the CPU emulation only so far.  The gene set is rebuilt on the device from the driver's -f file with
	// refSet's k, hitLenRequired and radius (main.cpp:766-771, 1082-1083); sortedReads[i].geneOverlap[0..3] receive what
	// AnnotateRead would have stored (an entry without a gene: seqIdx -1, strand 1).
	template <class Reads, class RefSet>
	bool BatchAnnotate( Reads &sortedReads, RefSet &refSet, int readCnt )
	{
		const char *env = getenv( "T4_ANNOTATE" ) ;
		if ( !gpu || env == NULL || atoi( env ) != 1 || getenv( "T4_STREAMS" ) == NULL || readCnt <= 0 || t4_adapter_ref_fa.empty() )
			return false ;
		t4_refset *ref = t4_refset_create_from_fa( t4_adapter_ref_fa.c_str(), refSet.kmerLength ) ;
		if ( !ref )
			Die() ;
		Check( t4_refset_set_hit_len_required( ref, refSet.hitLenRequired ) ) ;
		Check( t4_refset_set_radius( ref, refSet.radius ) ) ;
		const int ng = Check( t4_refset_size( ref ) ) ;
		bool same = ng == (int)refSet.seqs.size() ;
		for ( int i = 0 ; same && i < ng ; ++i )
			same = !strcmp( t4_refset_name( ref, i ), refSet.seqs[i].name ) ;
		if ( !same )
		{
			fprintf( stderr, "trust4_b200: the device gene set differs from the driver's (%d vs %d sequences)\n", ng, (int)refSet.seqs.size() ) ;
			exit( 1 ) ;
		}
		std::string pool ;
		std::vector<uint64_t> off( readCnt ) ;
		std::vector<int32_t> len( readCnt ) ;
		for ( int i = 0 ; i < readCnt ; ++i )
		{
			off[i] = pool.size() ;
			len[i] = (int)strlen( sortedReads[i].read ) ;
			if ( len[i] > T4_MAX_READ_LEN )
			{
				fprintf( stderr, "trust4_b200: read longer than %d bases\n", T4_MAX_READ_LEN ) ;
				exit( 1 ) ;
			}
			pool.append( sortedReads[i].read, len[i] ) ;
		}
		pool.append( 16, '\0' ) ;
		std::vector<int32_t> go( (size_t)readCnt * 32 ) ;
		std::vector<double> sim( (size_t)readCnt * 4 ) ;
		Check( t4_refset_annotate( ref, pool.data(), pool.size(), off.data(), len.data(), readCnt, go.data(), sim.data() ) ) ;
		int annotated = 0 ;
		for ( int i = 0 ; i < readCnt ; ++i )
		{
			bool any = false ;
			for ( int j = 0 ; j < 4 ; ++j )
			{
				const int32_t *o = &go[( (size_t)i * 4 + j ) * 8] ;
				struct _overlap g ; // _overlap(): seqIdx -1, strand 1 (what AnnotateRead leaves defined for a missing gene)
				if ( o[0] >= 0 )
				{
					g.seqIdx = o[0] ; g.readStart = o[1] ; g.readEnd = o[2] ; g.seqStart = o[3] ; g.seqEnd = o[4] ;
					g.strand = o[5] ; g.matchCnt = o[6] ; g.indelCnt = o[7] ;
					g.similarity = sim[(size_t)i * 4 + j] ;
					any = true ;
				}
				sortedReads[i].geneOverlap[j] = g ;
			}
			if ( any )
				++annotated ;
		}
		t4_refset_free( ref ) ;
		fprintf( stderr, "[trust4_b200] batch route: rough annotation on the device, %d of %d reads hit a gene\n", annotated, readCnt ) ;
		return true ;
	}

	int AddRead( char *read, char *geneName, int &strand, int barcode, int minKmerCount, bool repetitiveData, double similarityThreshold )
	{
		if ( !gpu )
			return SeqSet::AddRead( read, geneName, strand, barcode, minKmerCount, repetitiveData, similarityThreshold ) ;
		if ( replay )
		{
			if ( cur < bRet.size() ) // main loop, iteration `cur` (Size() closes an iteration)
			{
				if ( bEv[cur] & ( T4_EV_NOVEL_ANCHORED | T4_EV_NOVEL_MOTIF ) )
					return -1 ; // AddRead failed; the InputNovelRead that follows returns the recorded slot
				if ( bRet[cur] >= 0 )
					strand = bStrand[cur] ; // SeqSet.hpp:4469: only set on success
				return bRet[cur] ;
			}
			// rescue pass (main.cpp:1897-1940): reads with addRet == -2, in order
			if ( rescuePos >= rescueOrder.size() )
			{
				fprintf( stderr, "trust4_b200: replay out of step (rescue)\n" ) ;
				exit( 1 ) ;
			}
			int i = rescueOrder[rescuePos++] ;
			strand = bStrand[i] ;
			return bResc[i] ;
		}
		return Check( t4_seqset_add_read( h, read, geneName, &strand, barcode, minKmerCount, repetitiveData, similarityThreshold ) ) ;
	}
	int RepeatAddRead( char *read )
	{
		if ( gpu && replay && cur < bRet.size() )
			return bRet[cur] ;
		return gpu ? Check( t4_seqset_repeat_add_read( h, read ) ) : SeqSet::RepeatAddRead( read ) ;
	}
	int InputNovelRead( const char *id, char *read, int strand, int barcode )
	{
		if ( gpu && replay && cur < bRet.size() )
			return bRet[cur] ; // negative when the device loop made no such call (hint from a mate in another shard)
		return gpu ? Check( t4_seqset_input_novel_read( h, id, read, strand, barcode ) ) : SeqSet::InputNovelRead( id, read, strand, barcode ) ;
	}
	void UpdateAllConsensus()
	{
		if ( gpu && replay )
			return ; // done on the device (periodic, after the loop, after the rescue pass)
		if ( gpu ) Check( t4_seqset_update_all_consensus( h ) ) ; else SeqSet::UpdateAllConsensus() ;
	}
	void ChangeKmerLength( int kl )
	{
		if ( gpu && !replay )
			Check( t4_seqset_change_kmer_length( h, kl ) ) ;
		if ( gpu )
			curK = kl ;
		SeqSet::ChangeKmerLength( kl ) ; // keeps kmerLength of the CPU object in step (its seqs are empty until SyncToHost)
	}
	int Size()
	{
		if ( gpu && replay )
		{
			// main.cpp:1874 asks once per iteration: answer so that the driver's indexKmerLength follows the device's k
			int r = 0 ;
			if ( cur < bEv.size() && ( bEv[cur] & T4_EV_CHANGE_K ) && curK < maxFinalK )
				r = INT_MAX ;
			++cur ;
			return r ;
		}
		return gpu ? Check( t4_seqset_size( h ) ) : SeqSet::Size() ;
	}
	int SetHitLenRequired( int l )
	{
		if ( gpu )
		{
			Check( t4_seqset_set_hit_len_required( h, l ) ) ;
			curHitLen = l ;
		}
		return SeqSet::SetHitLenRequired( l ) ;
	}
	void SetIsLongSeqSet( bool in )
	{
		if ( gpu )
			Check( t4_seqset_set_is_long( h, in ) ) ;
		SeqSet::SetIsLongSeqSet( in ) ;
	}
	void SetConsiderBarcodeInIndexHash( bool s )
	{
		if ( gpu )
		{
			Check( t4_seqset_set_consider_barcode_in_hash( h, s ) ) ;
			curConsiderBarcode = s ? 1 : 0 ;
		}
		SeqSet::SetConsiderBarcodeInIndexHash( s ) ;
	}
	// main.cpp:1855 -- one finished barcode, removeFromIndex = true, earlyStop = true
	void ReleaseFinishedBarcodeSeq( std::map<int, int> barcodes, bool removeFromIndex, int contigMinCov, bool earlyStop )
	{
		if ( !gpu )
		{
			SeqSet::ReleaseFinishedBarcodeSeq( barcodes, removeFromIndex, contigMinCov, earlyStop ) ;
			return ;
		}
		if ( replay )
			return ; // purged inside the device loop (cfg.release_barcodes)
		if ( barcodes.size() != 1 || !removeFromIndex || !earlyStop )
		{
			fprintf( stderr, "trust4_b200: ReleaseFinishedBarcodeSeq is only supported as the stage-1 driver calls it\n" ) ;
			exit( 1 ) ;
		}
		Check( t4_seqset_release_finished_barcode( h, barcodes.begin()->first, contigMinCov ) ) ;
	}
	// main.cpp:1954 (--contigMinCov)
	void ReleaseShallowContigs( int minCov )
	{
		if ( gpu )
			for ( size_t i = 0 ; i < sets.size() ; ++i )
				Check( t4_seqset_release_shallow_contigs( sets[i], minCov ) ) ;
		else
			SeqSet::ReleaseShallowContigs( minCov ) ;
	}
	// main.cpp:711 (--debug-ns)
	void InputNovelFa( char *filename )
	{
		if ( gpu )
			Check( t4_seqset_input_novel_fa( h, filename ) ) ;
		else
			SeqSet::InputNovelFa( filename ) ;
	}
	void Output( FILE *fp, std::vector<std::string> *barcodeIntToStr = NULL )
	{
		if ( !gpu )
		{
			SeqSet::Output( fp, barcodeIntToStr ) ;
			return ;
		}
		if ( sets.size() > 1 )
		{
			// read-sharded run: the output is the concatenation of the streams' contig sets with global slot numbers
			SyncToHost() ;
			SeqSet::Output( fp, barcodeIntToStr ) ;
			return ;
		}
		std::vector<const char *> names ;
		if ( barcodeIntToStr )
			for ( size_t i = 0 ; i < barcodeIntToStr->size() ; ++i )
				names.push_back( barcodeIntToStr->at( i ).c_str() ) ;
		Check( t4_seqset_output( h, fp, barcodeIntToStr ? names.data() : NULL, (int)names.size() ) ) ;
		SyncToHost() ; // from here on the driver only reads the contigs (main.cpp:2049 InputSeqSet)
	}
} ;

// The first line of the batch route, inserted in front of the AddRead loop of main.cpp (integration/make_batch_main.py).
#define T4_BATCH_PREPARE() seqSet.BatchPrepare( sortedReads, refSet, readCnt, hasBarcode, keepMissingBarcode, trimLevel, firstReadLen, \
	constantGeneEnd, contigMinCov, changeKmerLengthThreshold )

// Opt-in (T4_SORT=1), in front of std::sort( sortedReads ) (main.cpp:1078); see BatchSort.
#define T4_BATCH_SORT() if ( !seqSet.BatchSort( sortedReads ) )

// Opt-in (T4_KMERSTATS=1), in front of the count-statistics loop (main.cpp:981); see BatchKmerStats.
#define T4_BATCH_KMERSTATS() if ( !seqSet.BatchKmerStats( sortedReads, readCnt, trimLevel, countMyself, contigMinCov > 0 ) )

// Opt-in (T4_BCSTATS=1), in front of `if (hasBarcode)` (main.cpp:1123); see BatchBarcodeStats.
#define T4_BATCH_BARCODE_STATS() if ( !seqSet.BatchBarcodeStats( sortedReads, readCnt, hasBarcode ) )

// The third line (opt-in, T4_ANNOTATE=1), in front of the rough annotation loop (main.cpp:1084); see BatchAnnotate.
#define T4_BATCH_ANNOTATE() if ( !seqSet.BatchAnnotate( sortedReads, refSet, readCnt ) )

// The second line of the batch route, in front of the AssignRead loop (main.cpp:2075); see BatchAssign.
#define T4_BATCH_ASSIGN() if ( !seqSet.BatchAssign( extendedSeq, assembledReads, assembledReadCnt ) )

#define SeqSet T4GpuSeqSet
#endif
