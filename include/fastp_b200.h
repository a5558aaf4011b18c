/*
 * fastp_b200.h -- C-ABI of the H100-native per-read FASTQ preprocessing hot path.
 *
 * This library replaces the worker body of the reference (OpenGene/fastp v1.3.6)
 *   bool SingleEndProcessor::processSingleEnd(ReadPack*, ThreadConfig*)   src/seprocessor.cpp:197-325
 *   bool PairEndProcessor::processPairEnd(ReadPack*, ReadPack*, ThreadConfig*)   src/peprocessor.cpp:362-708
 * i.e. the per-read operator chain
 *   Stats::statRead (pre)      src/stats.cpp:191-291
 *   Filter::trimAndCut         src/filter.cpp:68-207
 *   PolyX::trimPolyG           src/polyx.cpp:16-42
 *   OverlapAnalysis::analyze   src/overlapanalysis.cpp:17-146          (PE)
 *   statInsertSize             src/peprocessor.cpp:710-723             (PE)
 *   BaseCorrector::correctByOverlapAnalysis  src/basecorrector.cpp:16-83   (PE)
 *   AdapterTrimmer::trimByOverlapAnalysis    src/adaptertrimmer.cpp:17-46  (PE)
 *   AdapterTrimmer::trimBySequence / trimByMultiSequences  src/adaptertrimmer.cpp:48-157
 *   PolyX::trimPolyX           src/polyx.cpp:49-116
 *   max_len clip (Read::resize src/read.cpp:62-67)
 *   Filter::passFilter         src/filter.cpp:15-57
 *   FilterResult counters      src/filterresult.cpp:28-36,99-107,124-203
 *   Stats::statRead (post)
 *
 * The reference has no plugin/FFI boundary; the seam is those two private member
 * functions.  INTEGRATION.md shows the host shim a maintainer adds (stage ReadPacks
 * into the SoA batch below, call fp_process_*, unstage fp_read_result back into
 * Read::mSeq/mQuality, fill Stats/FilterResult from fp_counters_fetch).
 *
 * Plain C: pointers and sizes only.  Every function returns 0 on success or a
 * negative FP_E_* code; nothing calls exit().  Semantics are those of
 * `fastp --thread 1` (SURVEY.md App. C) unless fp_params.thread0_semantics == 0.
 */
#ifndef FASTP_B200_H
#define FASTP_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- verdict codes: src/common.h:43-51 ---- */
#define FP_PASS_FILTER         0
#define FP_FAIL_POLY_X         4
#define FP_FAIL_OVERLAP        8
#define FP_FAIL_N_BASE        12
#define FP_FAIL_LENGTH        16
#define FP_FAIL_TOO_LONG      17
#define FP_FAIL_QUALITY       20
#define FP_FAIL_COMPLEXITY    24
#define FP_FAIL_ADAPTER_DIMER 28
#define FP_FILTER_RESULT_TYPES 32

/* ---- error codes ---- */
#define FP_OK              0
#define FP_E_INVAL        -1   /* bad argument / unsupported parameter combination */
#define FP_E_CUDA         -2   /* CUDA runtime error (see fp_last_error)             */
#define FP_E_NOMEM        -3
#define FP_E_TOOLARGE     -4   /* batch larger than ctx capacity                       */
#define FP_E_UNSUPPORTED  -5   /* option the device path does not implement            */

/* ---- limits ---- */
#define FP_MAX_STRIDE       512   /* bytes per read row (multiple of 16)              */
#define FP_MAX_ADAPTER_LEN  255   /* per adapter sequence                             */
#define FP_MAX_ADAPTERS     512   /* r1 + r2 + fasta list                             */
#define FP_KMER_BINS       1024   /* 5-mers; reference allocates 2048 (stats.cpp:45), upper half stays 0 */
#define FP_QUAL_BINS        128   /* stats.h:85                                       */
#define FP_CYCLE_KINDS       34   /* Q30[8] Q20[8] content[8] qualsum[8] totalBase totalQual (stats.cpp:54-63) */

/* POD mirror of the Options fields the chain reads (src/options.h). */
typedef struct fp_params {
    int32_t paired;                 /* 0 = SE (processSingleEnd), 1 = PE (processPairEnd) */
    int32_t thread0_semantics;      /* 1: behave as worker thread 0 of `--thread 1`: overlap analysis + insert size on every pair
                                       (peprocessor.cpp:438,449,497). 0: as worker tid!=0.                                    */
    /* TrimmingOptions  options.h:223-246 */
    int32_t trim_front1, trim_tail1, trim_front2, trim_tail2, max_len1, max_len2;
    /* QualityCutOptions options.h:132-170 */
    int32_t cut_front, cut_tail, cut_right;
    int32_t cut_front_window, cut_front_quality;
    int32_t cut_tail_window,  cut_tail_quality;
    int32_t cut_right_window, cut_right_quality;
    /* PolyGTrimmerOptions / PolyXTrimmerOptions options.h:82-102 */
    int32_t polyg_enabled, polyg_min_len;
    int32_t polyx_enabled, polyx_min_len;
    /* AdapterOptions options.h:197-221 */
    int32_t adapter_enabled;
    int32_t has_seq_r1, has_seq_r2;         /* adapter.hasSeqR1 / hasSeqR2                     */
    const char* adapter_seq_r1;             /* adapter.sequence   (NUL terminated, may be NULL) */
    const char* adapter_seq_r2;             /* adapter.sequenceR2                               */
    int32_t n_fasta_adapters;               /* adapter.hasFasta <=> n_fasta_adapters > 0        */
    const char* const* fasta_adapters;      /* adapter.seqsInFasta                              */
    int32_t allow_gap_overlap_trimming;     /* --allow_gap_overlap_trimming (overlapanalysis.cpp:91) */
    int32_t dimer_max_len;                  /* adapter.dimerMaxLen (default 2)                  */
    /* CorrectionOptions + overlap thresholds options.h:123-130,376-379 (defaults 30/5/20 options.cpp:24-26) */
    int32_t correction_enabled;
    int32_t overlap_require, overlap_diff_limit, overlap_diff_percent_limit;
    /* QualityFilteringOptions options.h:248-268 */
    int32_t qual_filter_enabled;
    int32_t qualified_qual;                 /* ASCII char, num2qual(15) = '0' by default        */
    int32_t unqualified_percent_limit, n_base_limit, avg_qual_req;
    /* ReadLengthFilteringOptions options.h:270-284 */
    int32_t length_filter_enabled, length_required, length_limit;
    /* LowComplexityFilterOptions options.h:60-69 */
    int32_t complexity_filter_enabled;
    double  complexity_threshold;           /* int/100.0 as main.cpp:343 builds it              */
    /* insert size histogram  options.cpp:23, peprocessor.cpp:24-26 */
    int32_t insert_size_max;                /* default 512                                      */
    /* sequence lengths from the pre-scan (Options::seqLen1/2, options.h:366-367): Stats::mEvaluatedSeqLen */
    int32_t seq_len1, seq_len2;
    /* OverrepresentedSequenceAnasysOptions options.h:71-80 + the candidate lists the Evaluator pre-scan produced
     * (Options::overRepSeqs1/2, options.h:364-365; Evaluator::computeOverRepSeq evaluator.cpp:78-169 stays on the host).
     * Domain, as the Evaluator produces it: seq_len1/2 >= 2 (the fifth scan length is min(150, seq_len - 2)); each list free of
     * duplicates and of empty strings (the keys of a map), of any size, empty for one mate or both; reads may be longer or shorter
     * than seq_len (hit positions at or past seq_len are not counted in the dist). */
    int32_t overrep_enabled;
    int32_t overrep_sampling;               /* default 20 */
    int32_t n_overrep1;
    const char* const* overrep_seqs1;       /* keys of overRepSeqs1 (any order; the layout keeps this order) */
    int32_t n_overrep2;
    const char* const* overrep_seqs2;
    /* MergeOptions options.h:104-121 (PE only).  After the chain the pair is analysed again on the trimmed reads (peprocessor.cpp:521-523);
     * an overlapped pair becomes ONE read, r1[0, len1) + reverse complement of r2[0, len2) with len1 = overlap_len + max(0, offset),
     * len2 = offset > 0 ? len(r2) - overlap_len : 0 (OverlapAnalysis::merge, overlapanalysis.cpp:148-179); that read is filtered
     * (weight 2 in the FilterResult counters) and, when it passes, is what the post-filter Stats of read 1 see.  The post-filter Stats of
     * read 2 stay empty in this mode (peprocessor.cpp:588-591).  Records of a merged pair carry FP_F_MERGED, the merged read's verdict in
     * verdict / pair_verdict and the (trimmed) windows of r1 and r2; fp_ov_result holds the second analysis, from which len1 / len2 follow
     * (fp_merged_lens).  Size the counter block for merged reads: `cycles` of fp_ctx_create >= 2 * read length. */
    int32_t merge_enabled;                  /* --merge; main.cpp also forces correction_enabled (options.cpp:120-121): the caller's job */
    int32_t merge_include_unmerged;         /* --include_unmerged: pairs that did not merge are filtered read by read and both counted in read 1's post Stats */
} fp_params;

/* Fill with the reference's defaults: Options::Options() (options.cpp:9-32) + nested
 * ctors (options.h) + what main.cpp sets with no flags (length filter on, main.cpp:337). */
void fp_params_default(fp_params* p, int paired);

/* One batch of reads (SE) or read pairs (PE) in fixed-stride SoA form.
 * Row i of seq1 starts at seq1 + i*stride and holds len1[i] valid bytes.
 * Bytes in [len, stride) are ignored. seq/qual are MODIFIED IN PLACE by base correction. */
#define FP_B_INDEXED 0x1     /* fp_batch.flags: first_read_index holds the GLOBAL index of unit 0 of this batch */
#define FP_B_PACK2BIT 0x2    /* fp_batch.flags, host entry points only: the library's host threads (fp_set_host_threads) pack the bases to
                              * 2 bits (+ a list of the 'N's) chunk by chunk, overlapped with the copies, so that 0.25 instead of 1 byte
                              * per base crosses PCIe; qualities go up from the caller's rows as they are.  Rows must hold A/C/G/T/N only
                              * (else FP_E_UNSUPPORTED); results, corrected rows and patch lists are the same as without the flag. */
typedef struct fp_batch {
    int64_t   n;            /* reads (SE) or pairs (PE)                     */
    int32_t   stride;       /* multiple of 16, <= FP_MAX_STRIDE             */
    int32_t   flags;        /* FP_B_*                                        */
    uint8_t  *seq1, *qual1; /* [n][stride] bases (ASCII) / phred+33 quals    */
    uint16_t *len1;         /* [n]                                          */
    uint8_t  *seq2, *qual2; /* PE only                                      */
    uint16_t *len2;
    /* Position of unit 0 in the whole input stream (all batches, all ranks): the pre-filter over-representation
     * sampling test is `mReads % overRepSampling == 0` on that running count (src/stats.cpp:272).  Used only with
     * FP_B_INDEXED; without it the ctx continues its own count from the previous batch (single-process use). */
    int64_t   first_read_index;
} fp_batch;

/* flags */
#define FP_F_DROPPED          0x01  /* trimAndCut returned NULL (filter.cpp:78,101,134,170,196) */
#define FP_F_ADAPTER_TRIMMED  0x02  /* counted by incTrimmedAdapterRead                        */
#define FP_F_POLYX_TRIMMED    0x04  /* addPolyXTrimmed was called                              */
#define FP_F_CORRECTED        0x08  /* at least one base of this read was overwritten          */
#define FP_F_POLYG_TRIMMED    0x10  /* trimPolyG shortened the read                            */
#define FP_F_ADAPTER_DIMER    0x20
#define FP_F_MERGED           0x80  /* --merge: the pair overlapped and was merged (on both records); verdict = the merged read's */
#define FP_F_DUPLICATE        0x40  /* dedupOut: flagged by the duplicate filter with --dedup on; not written, not in the post-filter stats (peprocessor.cpp:397-401,575) */

typedef struct fp_read_result {
    uint16_t front;        /* frontTrimmed: bases removed at the 5' end by trimAndCut          */
    uint16_t len;          /* final length; the kept window is [front, front+len) of the input */
    uint8_t  verdict;      /* this read's passFilter code after the dimer override             */
    uint8_t  flags;        /* FP_F_*                                                           */
    int16_t  adapter_pos;  /* last trimBySequence hit position (trimmed coords; <0: A-tail skip), else 0 */
    uint16_t adapter_len;  /* adapter bases of this read added to mTrimmedAdapterBases         */
    uint8_t  polyx_base;   /* 0..3 = A,T,C,G (ATCG_BASES common.h:25); 255 = none              */
    uint8_t  pair_verdict; /* code passed to addFilterResult: SE = verdict, PE = max(r1,r2)    */
    uint16_t polyx_len;    /* bases removed by trimPolyX                                       */
    uint16_t reserved;
} fp_read_result;          /* 16 bytes */

/* mirror of OverlapResult src/overlapanalysis.h:15-22 */
typedef struct fp_ov_result {
    uint8_t overlapped, has_gap;
    int16_t offset, overlap_len, diff;
} fp_ov_result;            /* 8 bytes */

/* --merge: the two pieces of a merged read (OverlapAnalysis::merge, overlapanalysis.cpp:149-157): merged = r1[0, len1) followed by the
 * reverse complement of r2[0, len2), both in TRIMMED coordinates (add fp_read_result.front for the row index); r2_len = out2.len. */
static inline void fp_merged_lens(const fp_ov_result* ov, int r2_len, int* len1, int* len2) {
    *len1 = ov->overlap_len + (ov->offset > 0 ? ov->offset : 0);
    *len2 = ov->offset > 0 ? r2_len - ov->overlap_len : 0;
}

/* A base overwritten by BaseCorrector (basecorrector.cpp:44-60). */
typedef struct fp_patch {
    uint32_t pair;         /* index in the batch                 */
    uint16_t pos;          /* position in the ORIGINAL read row  */
    uint8_t  which;        /* 0 = read1, 1 = read2               */
    uint8_t  base;         /* new base                           */
    uint8_t  qual;         /* new quality                        */
    uint8_t  old_base;     /* what the row held before (lets a caller that keeps its batch resident undo the pass) */
    uint8_t  old_qual;
    uint8_t  _pad;
} fp_patch;                /* 12 bytes */

/* One call of FilterResult::addAdapterTrimmed (src/filterresult.cpp:124-180) as the chain made it -- the adapter STRINGS the reference
 * histograms (`adapter_cutting.read1_adapter_counts` of the JSON report) are substrings of the read rows or prefixes of the configured
 * adapters, so the device records where they are and the host rebuilds the maps in input order with the reference's own caps
 * (MAX_ADAPTER_REC / LOW_COMPLEXITY_SKIP are applied in arrival order, src/filterresult.cpp:7-8,135).  Events are appended to the list
 * in no particular order: sort by (unit, key).  Within a unit the calls come in the order of `key`.
 *   FP_EV_PAIR    trimByOverlapAnalysis (src/adaptertrimmer.cpp:17-46): addAdapterTrimmed(adapter1, adapter2) -- two events of one unit
 *                 (which = 0 and 1, len may be 0); the string is row[start, start+len) of that read (current, i.e. corrected, bytes)
 *   FP_EV_READ    trimBySequence hit at pos >= 0 (:147-152): addAdapterTrimmed(row[start, start+len), isR2 = which)
 *   FP_EV_ADAPTER trimBySequence hit at pos < 0 (:139-146): the string is the first `len` bases of adapter number `adapter`
 *                 (0 = adapter_seq_r1, 1 = adapter_seq_r2, 2+i = fasta_adapters[i])                                            */
#define FP_EV_PAIR    0
#define FP_EV_READ    1
#define FP_EV_ADAPTER 2
typedef struct fp_adapter_event {
    uint32_t unit;         /* index in the batch (host entry points: in the whole host batch) */
    uint16_t start, len;
    uint16_t key;          /* order of the calls inside one unit */
    uint8_t  which;        /* 0 = read1, 1 = read2 */
    uint8_t  kind;         /* FP_EV_* */
    uint16_t adapter;      /* FP_EV_ADAPTER: which adapter */
    uint16_t _pad;
} fp_adapter_event;        /* 16 bytes */

/* ---------------- packed counter block (all int64, plain sums) ----------------
 * stats[s], s in {0:pre1, 1:post1, 2:pre2, 3:post2}  (SE uses 0,1):
 *     cycle[34][C]   kinds in the reference's order (stats.cpp:54-63); slot = base & 7
 *     kmer[1024]     code = base-4 digits A0 T1 C2 G3, first base most significant (stats.cpp:228-266)
 *     qualhist[128]  indexed by the raw quality char (stats.cpp:213)
 *     reads, lengthSum (stats.cpp:194,290)
 * filter:  filterReadStats[32] | trimmedAdapterRead | trimmedAdapterBases | polyXReads[4] | polyXBases[4]
 *          | correction[64] | correctedReads | mergedPairs          (filterresult.h:66-79)
 * isize:   insertSizeHist[insert_size_max+1]                          (peprocessor.cpp:24-26)
 */
#define FP_STATS_PRE1  0
#define FP_STATS_POST1 1
#define FP_STATS_PRE2  2
#define FP_STATS_POST2 3

typedef struct fp_counter_layout {
    int32_t cycles;        /* C: capacity of the per-cycle arrays (>= longest read)   */
    int32_t n_stats;       /* 2 (SE) or 4 (PE)                                        */
    int32_t isize_bins;    /* insert_size_max + 1                                     */
    int32_t _pad;
    int64_t stats_stride;  /* int64 words per Stats block                             */
    int64_t off_kmer, off_qualhist, off_reads, off_length_sum;   /* inside a Stats block */
    int64_t off_filter;    /* start of the FilterResult block                         */
    int64_t off_isize;     /* start of the insert-size histogram                      */
    /* over-representation (stats.cpp:270-288): per Stats s: count[K_s] then dist[K_s][seqLen_s]; K/seqLen per SIDE */
    int32_t n_overrep[2];  /* candidates of read1 / read2                             */
    int32_t overrep_len[2];/* mEvaluatedSeqLen of read1 / read2                       */
    int64_t off_overrep[4];/* start of each Stats' over-representation region         */
    int64_t total;         /* total int64 words                                       */
} fp_counter_layout;

/* offsets inside the FilterResult block */
#define FP_FR_READSTATS        0
#define FP_FR_ADAPTER_READS   32
#define FP_FR_ADAPTER_BASES   33
#define FP_FR_POLYX_READS     34
#define FP_FR_POLYX_BASES     38
#define FP_FR_CORRECTION      42
#define FP_FR_CORRECTED_READS 106
#define FP_FR_MERGED_PAIRS    107
#define FP_FR_WORDS           108

void fp_counter_layout_make(fp_counter_layout* L, int paired, int cycles, int insert_size_max);
/* same, with over-representation regions for k1/k2 candidates and evaluated sequence lengths len1/len2 */
void fp_counter_layout_make_overrep(fp_counter_layout* L, int paired, int cycles, int insert_size_max, int k1, int len1, int k2, int len2);
/* ABI self-check for bindings: sizeof of 0:fp_params 1:fp_batch 2:fp_read_result 3:fp_ov_result 4:fp_patch 5:fp_counter_layout */
size_t fp_abi_sizeof(int which);

#ifdef __CUDACC__
#define FP_INLINE static __host__ __device__ __forceinline__
#else
#define FP_INLINE static inline
#endif
FP_INLINE int64_t fp_off_cycle(const fp_counter_layout* L, int stats, int kind, int cycle) {
    return (int64_t)stats * L->stats_stride + (int64_t)kind * L->cycles + cycle;
}
FP_INLINE int64_t fp_off_kmer(const fp_counter_layout* L, int stats, int code) {
    return (int64_t)stats * L->stats_stride + L->off_kmer + code;
}
FP_INLINE int64_t fp_off_qualhist(const fp_counter_layout* L, int stats, int q) {
    return (int64_t)stats * L->stats_stride + L->off_qualhist + q;
}
FP_INLINE int64_t fp_off_reads(const fp_counter_layout* L, int stats) {
    return (int64_t)stats * L->stats_stride + L->off_reads;
}
FP_INLINE int64_t fp_off_length_sum(const fp_counter_layout* L, int stats) {
    return (int64_t)stats * L->stats_stride + L->off_length_sum;
}
FP_INLINE int64_t fp_off_overrep_count(const fp_counter_layout* L, int stats, int k) {
    return L->off_overrep[stats] + k;
}
FP_INLINE int64_t fp_off_overrep_dist(const fp_counter_layout* L, int stats, int k, int pos) {
    const int side = stats >> 1;
    return L->off_overrep[stats] + L->n_overrep[side] + (int64_t)k * L->overrep_len[side] + pos;
}

/* ---------------- device context ---------------- */
typedef struct fp_ctx fp_ctx;

/* Create a context on CUDA device `device` for batches of up to max_batch reads/pairs of
 * `stride` bytes per row; per-cycle counters cover `cycles` cycles (>= longest read).
 * Fails with FP_E_CUDA if no usable device / the CUDA kernels cannot be loaded: there is no CPU fallback. */
int  fp_ctx_create(const fp_params* p, int device, int64_t max_batch, int32_t stride, int32_t cycles, fp_ctx** out);
void fp_ctx_destroy(fp_ctx* ctx);
const char* fp_last_error(void);

int  fp_ctx_layout(const fp_ctx* ctx, fp_counter_layout* out);

/* HBM-resident entry points: every pointer in `b`, and out1/out2/ov/patches, is DEVICE memory on the
 * ctx's device. Work is enqueued on `stream` (a cudaStream_t passed as void*; NULL = the ctx's own
 * stream) and NOT synchronised. Counters accumulate inside the ctx until fp_counters_reset.
 * ov / patches / n_patches may be NULL.  patches capacity = patch_cap entries; *n_patches counts all
 * corrections (may exceed patch_cap: extra ones are applied in place but not listed).               */
int  fp_process_se(fp_ctx* ctx, const fp_batch* b, fp_read_result* out1, void* stream);
int  fp_process_pe(fp_ctx* ctx, const fp_batch* b, fp_read_result* out1, fp_read_result* out2,
                   fp_ov_result* ov, fp_patch* patches, uint32_t patch_cap, uint32_t* n_patches, void* stream);

/* Host-buffer entry points (the call the reference-side shim makes): every pointer is HOST memory
 * (pinned or pageable).  b->stride is the HOST row pitch here: any value from the longest read up to the ctx stride (a pitch equal to the
 * read length sends no padding bytes over PCIe; the rows are re-pitched in HBM). Copies inputs H2D in chunks on two streams, runs the kernels, copies the
 * per-read records back and applies base-correction patches to the host seq/qual rows. Synchronous. */
int  fp_process_se_host(fp_ctx* ctx, const fp_batch* b, fp_read_result* out1);
int  fp_process_pe_host(fp_ctx* ctx, const fp_batch* b, fp_read_result* out1, fp_read_result* out2,
                        fp_ov_result* ov);
/* Same, and the base corrections it applied to the host rows are also listed for the caller (HOST array of patch_cap entries,
 * fp_patch.pair = index in `b`; *n_patches counts all of them and may exceed patch_cap): the reference-side shim uses it to
 * touch only the Read objects whose bases changed (BaseCorrector rewrites r1/r2 in place, src/basecorrector.cpp:44-60).
 * Internally a host chunk (up to 262144 pairs) lists at most 2 per pair + 1024 corrections.  A chunk with more still gets its
 * corrected rows written back whole, but the list cannot be complete: *n_patches is then at least 2^63 - 1.          */
int  fp_process_pe_host_patches(fp_ctx* ctx, const fp_batch* b, fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov,
                                fp_patch* patches, uint64_t patch_cap, uint64_t* n_patches);

/* Adapter-string events (above).  Device form: `events` (capacity `cap`) and `count` are DEVICE memory that later fp_process_se / _pe
 * calls append to (*count keeps counting past cap; the caller zeroes it); NULL switches the recording off (the default).
 * Host form: the fp_process_*_host calls append to a HOST array with fp_adapter_event.unit relative to the host batch and set
 * *n_events (which may exceed cap) -- what the reference-side shim feeds to FilterResult::addAdapterTrimmed after sorting by (unit, key).
 * A host chunk buffers 2 + 2 * n_fasta_adapters events per pair (1 + n_fasta_adapters per read), the most the chain can make, up to
 * 2^24 per chunk; a chunk that makes more (possible only beyond 30 fasta adapters PE, 62 SE) fails the call with FP_E_TOOLARGE. */
int  fp_set_event_sink(fp_ctx* ctx, fp_adapter_event* d_events, uint32_t cap, uint32_t* d_count);
int  fp_set_host_event_sink(fp_ctx* ctx, fp_adapter_event* h_events, uint64_t cap, uint64_t* n_events);
/* Host threads the library may use for FP_B_PACK2BIT (the reference's counterpart is its `-w` worker count, src/options.h:thread).
 * 0 (the default) = the CPUs this process can really use (affinity mask, cgroup quota) minus one. */
int  fp_set_host_threads(fp_ctx* ctx, int threads);

/* ---------------- packed host rows: the end-to-end path is PCIe-bound, so send fewer bytes ----------------
 * 2 bits per base (code = (ascii >> 1) & 3: A0 C1 T2 G3; base k of a read in bits 2(k&3) of byte k>>2), qualities as they are, rows at
 * the caller's pitch (no padding to the device stride), 'N' positions as a sorted exception list: 2x150 bp -> about 385 bytes per
 * pair instead of 644.  fp_host_pack_rows packs host SoA rows with `threads` host threads (word-at-a-time fast path for runs of
 * A/C/G/T; FP_E_UNSUPPORTED if a base outside {A,C,G,T,N} turns up -- send that batch through fp_process_*_host instead).
 * fp_process_*_host_packed = fp_process_*_host on packed input: H2D of the packed arrays, a small kernel restores the stride rows in
 * HBM, then the same chain.  The packed buffers are never modified; base corrections come back as the patch list only.  When a host
 * chunk makes more corrections than its internal list holds (above) the library cannot list them all; if the caller asked for the list
 * (n_patches != NULL) fp_process_pe_host_packed then fails with FP_E_TOOLARGE (records and counters of the chunks before it are
 * already written).  fp_process_pe_host / _patches write corrected rows back instead and have no such limit.                 */
typedef struct fp_npos { uint32_t unit; uint16_t pos; uint8_t which; uint8_t _pad; } fp_npos;   /* base `pos` of read `which` of unit `unit` is 'N' */
typedef struct fp_packed_batch {
    int64_t   n;
    int32_t   pitch_b, pitch_q;     /* bytes per read in bases* / qual* (pitch_b >= (longest read + 3) / 4, pitch_q >= longest read) */
    uint8_t  *bases1, *qual1;       /* [n][pitch_b], [n][pitch_q] */
    uint16_t *len1;
    uint8_t  *bases2, *qual2;       /* PE only */
    uint16_t *len2;
    fp_npos  *npos;                 /* sorted by unit */
    int64_t   n_npos, npos_cap;
    int32_t   flags;                /* FP_B_INDEXED as in fp_batch */
    int32_t   _pad;
    int64_t   first_read_index;
} fp_packed_batch;
int  fp_host_pack_rows(const fp_batch* rows, int paired, fp_packed_batch* out, int threads);
int  fp_process_se_host_packed(fp_ctx* ctx, const fp_packed_batch* pb, fp_read_result* out1);
int  fp_process_pe_host_packed(fp_ctx* ctx, const fp_packed_batch* pb, fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov,
                               fp_patch* patches, uint64_t patch_cap, uint64_t* n_patches);

/* Counter block. fetch synchronises the ctx's streams, finalises (totals per cycle) and copies
 * layout.total int64 words to host_out. */
int  fp_counters_reset(fp_ctx* ctx);
int  fp_counters_fetch(fp_ctx* ctx, int64_t* host_out);
/* Device pointer to the RAW int64 block (layout.total words; the per-cycle totals, kinds 32/33, are derived from it by
 * fp_counters_fetch) for an in-place ncclAllReduce(ncclInt64, ncclSum) / torch.distributed.all_reduce by the caller
 * (Stats::merge src/stats.cpp:877-955 and FilterResult::merge src/filterresult.cpp:38-89 are element-wise sums).
 * After the all-reduce the block holds the job's totals: fetch it, then fp_counters_reset before processing more --
 * reducing twice, or processing on top of a reduced block, counts the other ranks' reads again. */
int  fp_counters_device_ptr(fp_ctx* ctx, int64_t** dev_ptr, int64_t* n_words);
/* Collective form: `comm` is an ncclComm_t (void*); no-op when comm == NULL.  Enqueued on `stream` (NULL = the ctx's own)
 * after everything already enqueued there, not synchronised: fp_counters_fetch waits for it. */
int  fp_counters_allreduce(fp_ctx* ctx, void* comm, void* stream);

/* Undo the base corrections of one fp_process_pe pass on a batch that stays resident in DEVICE memory: writes old_base /
 * old_qual of the first n_patches entries of `patches` (device memory, as filled by that pass) back into the rows.
 * A position is corrected at most once per pass, so the order of the list does not matter. */
int  fp_patches_undo(fp_ctx* ctx, const fp_batch* b, const fp_patch* patches, const uint32_t* n_patches, uint32_t patch_cap, void* stream);

/* ---- over-representation sampling across batches / ranks (SURVEY.md 8(e), src/stats.cpp:270-290) ----
 * PRE-filter stats sample unit i iff (global index of i) % sampling == 0: pass fp_batch.first_read_index (FP_B_INDEXED).
 * POST-filter stats sample by the running count of reads that PASSED before this one in the whole stream, which a rank
 * only knows once every earlier shard has been filtered.  Two-phase protocol for sharded runs:
 *   fp_overrep_defer_post(ctx, 1)     the fp_process_* calls skip the post-filter scan
 *   fp_pass_count(...)                units of a processed batch that were counted by the post-filter Stats
 *   (exclusive scan of the counts over batches and ranks -- one int64 per rank through ncclAllGather / all_gather)
 *   fp_overrep_post(..., pass_base)   post-filter scan of that batch given the number of counted units before it
 * out1/out2 are the DEVICE record arrays the fp_process_* call filled for that batch; the batch rows must still hold
 * what that call left (corrected bases included). */
int  fp_overrep_defer_post(fp_ctx* ctx, int32_t defer);
int  fp_pass_count(fp_ctx* ctx, const fp_read_result* out1, int64_t n, int64_t* count, void* stream);   /* synchronises `stream` */
int  fp_overrep_post(fp_ctx* ctx, const fp_batch* b, const fp_read_result* out1, const fp_read_result* out2, int64_t pass_base, void* stream);

/* ---------------- FASTQ text <-> rows on the device (SURVEY.md 8(f) rank 1) ----------------
 * fp_fastq_decode  replaces FastqReader::read / getLine (src/fastqreader.cpp:240-368) for a chunk of plain FASTQ text that
 *                  is already in DEVICE memory: it finds the records, checks them like the reference ('+' line, equal
 *                  lengths) and scatters bases / qualities into rows of `stride` bytes (zero-filled behind the read).
 * fp_fastq_encode  replaces Read::appendToString (src/read.cpp:119-134) for the reads / pairs that pass
 *                  (src/peprocessor.cpp:583-584, src/seprocessor.cpp:268): name, trimmed (and corrected) bases, strand line,
 *                  trimmed qualities, in input order.
 * Line rules are the reference's: '\n', or a '\r' not followed by '\n', ends a line; "\r\n" is one terminator; a record starts
 * at the first non-empty line beginning with '@'; the next three lines are taken as they come.  Where the reference reader
 * gives up (strand line not '+', lengths differ) it stops reading: info->error / error_record say so and n_records counts
 * the records before it.  Chunks must be smaller than 4 GiB.                                                             */
#define FP_FQ_OK            0
#define FP_FQ_ERR_STRAND    1   /* "Expected '+'"  fastqreader.cpp:349  */
#define FP_FQ_ERR_LENGTH    2   /* sequence and quality have different length  fastqreader.cpp:356 */
#define FP_FQ_ERR_STRIDE    3   /* a read is longer than the row stride (not a reference error) */
typedef struct fp_fastq_rec { uint32_t name_off, name_len, strand_off, strand_len; } fp_fastq_rec;   /* offsets into the chunk */
typedef struct fp_fastq_info {
    int64_t n_records;      /* records decoded into the rows (<= capacity)                              */
    int64_t consumed;       /* bytes of the chunk they cover (the caller carries the rest to the next chunk) */
    int64_t n_lines;        /* lines seen in the chunk                                                  */
    int32_t error;          /* FP_FQ_* of the first bad record, FP_FQ_OK if none                        */
    int32_t more;           /* 1 if complete records were left because capacity was reached             */
    int64_t error_record;   /* its index, -1 if none                                                    */
} fp_fastq_info;
/* d_text .. d_recs are DEVICE pointers; final_chunk: the text ends here (an unterminated last line counts).  Synchronous. */
int  fp_fastq_decode(fp_ctx* ctx, const uint8_t* d_text, int64_t nbytes, int32_t final_chunk, int32_t phred64,
                     uint8_t* d_seq, uint8_t* d_qual, uint16_t* d_len, int64_t capacity, fp_fastq_rec* d_recs,
                     fp_fastq_info* info);
/* Output text of side `d_res` (its pair_verdict decides, so for pairs both sides keep the same records).
 * *out_bytes = size of the full output; if it exceeds out_cap nothing beyond out_cap is written.  Synchronous. */
int  fp_fastq_encode(fp_ctx* ctx, const uint8_t* d_text, const fp_fastq_rec* d_recs, const fp_read_result* d_res,
                     const uint8_t* d_seq, const uint8_t* d_qual, int64_t n, uint8_t* d_out, int64_t out_cap, int64_t* out_bytes);
/* Whole path on HOST buffers: text chunk(s) in, filtered text out (text2/out2 NULL for single-end).
 * The chunk is worked through in rounds of at most the ctx's max_batch records: the text goes up in pieces on its own
 * stream while earlier pieces are decoded, run through the operator chain and encoded, and their output text goes down
 * on a third stream (pinned host buffers overlap; pageable ones work, serialised).  n_units = reads / pairs processed
 * (pairs end with the shorter side); consumed1/2 = bytes of each input they cover -- the caller prepends the rest
 * (an incomplete last record, the longer side's surplus) to its next chunk; final_chunk: no more input follows.
 * info1/2 (optional): records, lines, first reader error (the stream ends there, like FastqReader returning NULL).
 * Counters accumulate in the ctx as with fp_process_*.  Synchronous.                                            */
int  fp_fastq_process_host(fp_ctx* ctx, const uint8_t* text1, int64_t nbytes1, const uint8_t* text2, int64_t nbytes2,
                           int32_t final_chunk, int32_t phred64,
                           uint8_t* out1, int64_t out_cap1, int64_t* out_bytes1,
                           uint8_t* out2, int64_t out_cap2, int64_t* out_bytes2,
                           int64_t* n_units, int64_t* consumed1, int64_t* consumed2, fp_fastq_info* info1, fp_fastq_info* info2);

/* Merging mode (--merge, fp_params.merge_enabled) writes three streams, decided per pair from its two records (src/peprocessor.cpp:519-622):
 *   merged pair (FP_F_MERGED): if the merged read passes, ONE record on the merged stream, whatever the duplicate flag says (:528-534) --
 *       read 1's name line + " merged_<len1>_<len2>", r1[0, len1) + reverse complement of r2[0, len2) (fp_merged_lens; complement as
 *       src/simd.cpp:296-308: A<->T, C<->G in either case -> upper case, anything else -> 'N'), read 1's strand line (with the same suffix
 *       unless it is exactly "+"), q1[0, len1) + q2[0, len2) reversed (OverlapAnalysis::merge, src/overlapanalysis.cpp:148-179);
 *   not merged, --include_unmerged, neither read dropped: read 1 on the merged stream if its own verdict passes and the pair is not a
 *       flagged duplicate, then read 2 likewise (:537-556);
 *   every other pair: both reads to their sides under the ordinary rule (pair verdict passes, not a duplicate; :575-584).
 * fp_fastq_encode_merge writes ONE of the streams of a batch the chain has worked on (fp_process_pe with `ov`), all pointers DEVICE:
 *   which                FP_FQ_OUT_MERGED (--merged_out), FP_FQ_OUT_R1 (--out1) or FP_FQ_OUT_R2 (--out2)
 *   d_text1/2, d_recs1/2 the chunks fp_fastq_decode read and the records it wrote, per side (name and strand lines are copied from there)
 *   d_res1/2, d_ov       what fp_process_pe wrote: records of both reads and the second overlap analysis (:523) of every pair
 *   d_seq1/2, d_qual1/2  the rows as the chain left them (corrected bases included), ctx stride
 *   n, d_out, out_cap, out_bytes  as fp_fastq_encode: *out_bytes = size of the whole stream; a record that does not fit under out_cap
 *                        is left out whole.
 * FP_E_INVAL on a single-end ctx or one created without merge_enabled.  Synchronous. */
#define FP_FQ_OUT_MERGED 0
#define FP_FQ_OUT_R1     1
#define FP_FQ_OUT_R2     2
int  fp_fastq_encode_merge(fp_ctx* ctx, int32_t which, const uint8_t* d_text1, const fp_fastq_rec* d_recs1, const uint8_t* d_text2, const fp_fastq_rec* d_recs2,
                           const fp_read_result* d_res1, const fp_read_result* d_res2, const fp_ov_result* d_ov,
                           const uint8_t* d_seq1, const uint8_t* d_qual1, const uint8_t* d_seq2, const uint8_t* d_qual2,
                           int64_t n, uint8_t* d_out, int64_t out_cap, int64_t* out_bytes);
/* fp_fastq_process_host for a ctx that merges pairs: the same rounds, with the merged stream as a third host output (NULL = not wanted,
 * like out1 / out2).  With fp_fastq_set_dedup a merged read is written whatever its flag says; the other two cases honour it.
 * fp_fastq_process_host itself refuses such a ctx (FP_E_INVAL, nothing touched): its two outputs cannot hold what merging writes.
 * Create the ctx with cycles >= 2 * stride (fp_params.merge_enabled).  FP_E_INVAL on a ctx without merge_enabled. */
int  fp_fastq_process_host_merge(fp_ctx* ctx, const uint8_t* text1, int64_t nbytes1, const uint8_t* text2, int64_t nbytes2,
                                 int32_t final_chunk, int32_t phred64,
                                 uint8_t* out1, int64_t out_cap1, int64_t* out_bytes1,
                                 uint8_t* out2, int64_t out_cap2, int64_t* out_bytes2,
                                 uint8_t* merged, int64_t merged_cap, int64_t* merged_bytes,
                                 int64_t* n_units, int64_t* consumed1, int64_t* consumed2, fp_fastq_info* info1, fp_fastq_info* info2);

/* Reads that do not go to out1 / out2: --unpaired1, --unpaired2 and --failed_out (src/seprocessor.cpp:280-290, src/peprocessor.cpp:575-620).
 * Only a unit that is not a flagged duplicate and, in merging mode, took neither merging branch (not merged, not covered by
 * --include_unmerged) writes here.  A read "passes" when trimAndCut kept it and its own verdict (after the adapter-dimer override) is
 * FP_PASS_FILTER.  Single-end: a read that does not pass goes to failed, tagged with its reason.  Paired-end, by the writers that exist:
 *   both pass, or neither (an adapter-dimer pair is one of these): nothing here;
 *   only read 1 passes: with an unpaired-1 writer, read 1 to unpaired1 and read 2 to failed with its reason; without one, failed gets
 *       read 1 tagged "paired_read_is_failing", then read 2 with its reason;
 *   only read 2 passes: with an unpaired-2 writer, read 2 to unpaired2 and read 1 to failed with its reason; otherwise, with an unpaired-1
 *       writer, read 2 to unpaired1 and read 1 to failed; otherwise failed gets read 1 with its reason, then read 2 tagged
 *       "paired_read_is_failing".
 * A failed record is Read::appendToStringWithTag (src/read.cpp:136-154): the name line, ' ', the tag of FAILED_TYPES (src/common.h:56-65:
 * failed_too_many_n_bases, failed_too_short, failed_too_long, failed_quality_filter, failed_low_complexity, failed_adapter_dimer),
 * then sequence, strand and quality lines.  The read written is the one trimAndCut changed in place: its kept window with any corrected
 * bases; a read trimAndCut dropped (FP_F_DROPPED) was never touched and is written whole, row bytes [0, decoded length).  Unpaired
 * records are written like out1 / out2.  A tagged record is at most 24 bytes longer than the input record.
 * Writers: the reference's --unpaired2 defaults to --unpaired1 and is a writer of its own only when the two names differ
 * (src/main.cpp:188-189, src/peprocessor.cpp:68-72).  Its CLI hands the unpaired-2 text to a file only when both writers exist (:681-686);
 * the library returns it whenever FP_FQ_W_UNPAIRED2 is set and leaves that choice to the caller.
 * fp_fastq_encode_rejects writes ONE stream of a batch the chain has worked on, all pointers DEVICE (side 2 NULL for single-end):
 *   which                FP_FQ_OUT_UNPAIRED1 / _UNPAIRED2 (paired only) or FP_FQ_OUT_FAILED
 *   writers              FP_FQ_W_* of the unpaired writers that exist (0 for single-end)
 *   d_text*, d_recs*     as fp_fastq_encode_merge; d_res* what fp_process_se / _pe wrote (the merging branch is read off FP_F_MERGED)
 *   d_seq*, d_qual*      the rows as the chain left them; d_len* the decoded lengths (fp_fastq_decode's d_len; the chain does not change them)
 *   n, d_out, out_cap, out_bytes  as fp_fastq_encode.
 * FP_E_INVAL: unpaired stream or writers on a single-end ctx, writers on a ctx with merge_enabled and merge_include_unmerged (the reference
 * ignores both options there, src/options.cpp:136-143,222-229).  Synchronous. */
#define FP_FQ_OUT_UNPAIRED1 3
#define FP_FQ_OUT_UNPAIRED2 4
#define FP_FQ_OUT_FAILED    5
#define FP_FQ_OUTS          6
#define FP_FQ_W_UNPAIRED1   0x1
#define FP_FQ_W_UNPAIRED2   0x2
int  fp_fastq_encode_rejects(fp_ctx* ctx, int32_t which, int32_t writers, const uint8_t* d_text1, const fp_fastq_rec* d_recs1,
                             const uint8_t* d_text2, const fp_fastq_rec* d_recs2, const fp_read_result* d_res1, const fp_read_result* d_res2,
                             const uint8_t* d_seq1, const uint8_t* d_qual1, const uint16_t* d_len1,
                             const uint8_t* d_seq2, const uint8_t* d_qual2, const uint16_t* d_len2,
                             int64_t n, uint8_t* d_out, int64_t out_cap, int64_t* out_bytes);
/* The text path with every output stream: outs / out_caps / out_bytes are indexed by FP_FQ_OUT_* (merged, out1, out2, unpaired1, unpaired2,
 * failed).  A NULL buffer is not wanted; a NULL unpaired buffer also means that writer does not exist, which decides where reads go (above).
 * Works for single-end, paired and merging ctxs; out_bytes[k] is set for every k.  FP_E_INVAL, touching nothing: an unpaired buffer on a
 * single-end ctx or with merge_include_unmerged, a merged buffer on a ctx that does not merge, an out2 buffer on a single-end ctx.
 * FP_E_TOOLARGE when a stream outgrows its buffer, as for fp_fastq_process_host.  Everything else is fp_fastq_process_host(_merge). */
int  fp_fastq_process_host_outs(fp_ctx* ctx, const uint8_t* text1, int64_t nbytes1, const uint8_t* text2, int64_t nbytes2,
                                int32_t final_chunk, int32_t phred64, uint8_t* const outs[FP_FQ_OUTS], const int64_t out_caps[FP_FQ_OUTS],
                                int64_t out_bytes[FP_FQ_OUTS], int64_t* n_units, int64_t* consumed1, int64_t* consumed2,
                                fp_fastq_info* info1, fp_fastq_info* info2);

/* Interleaved pairs (--interleaved_in, --stdout): mates alternate in one text, read 1 then read 2 (FastqReaderPair::read with
 * interleaved = true, src/fastqreader.cpp:452-460).  The pair stream ends at the first record either mate's reader rejects (ReadPair::eof,
 * src/read.cpp:203-205): a rejected mate 2 also drops the good mate 1 before it, and a lone last record is dropped without a message.
 * fp_fastq_decode_interleaved is fp_fastq_decode for such a chunk: record r goes to side (r & 1), row (r >> 1), rows / lengths / records per
 * side (all DEVICE).  capacity and info->n_records count PAIRS; info->error_record is the first bad record's index among the chunk's
 * records (mates counted one by one).  A chunk that is not final and ends with a lone mate 1 is consumed up to that record's name line;
 * a final one drops it and is consumed whole.  Capacity cuts after record 2 * capacity.  Synchronous.
 * fp_fastq_encode_interleaved writes the --stdout stream of a paired ctx (src/peprocessor.cpp:579-581, singleOutput): for every pair,
 * read 1's record as fp_fastq_encode writes it on out1, then read 2's as it writes it on out2 -- byte for byte the two streams interleaved
 * record by record.  Arguments as fp_fastq_encode_merge (side 2's text may be side 1's).  FP_E_INVAL on a single-end ctx and on a ctx that
 * merges pairs (its stdout stream is the merged one: fp_fastq_encode_merge with FP_FQ_OUT_MERGED).  Synchronous.
 * fp_fastq_set_interleaved switches the text path (fp_fastq_process_host, _merge, _outs); both default to 0:
 *   in = 1   text1 holds both mates: pass text2 NULL and nbytes2 0; *consumed2 is 0 and *info2 is zeroed, info1 counts pairs.
 *   out = 1  the FP_FQ_OUT_R1 buffer (out1) receives the interleaved stream; an FP_FQ_OUT_R2 buffer (out2) is refused.
 * FP_E_INVAL, nothing changed: `in` on a single-end ctx, `out` on a single-end ctx or one that merges pairs.  The round loop itself refuses
 * (FP_E_INVAL, nothing touched) text2 / nbytes2 with `in`, and an out2 buffer with `out`. */
int  fp_fastq_decode_interleaved(fp_ctx* ctx, const uint8_t* d_text, int64_t nbytes, int32_t final_chunk, int32_t phred64,
                                 uint8_t* d_seq1, uint8_t* d_qual1, uint16_t* d_len1, fp_fastq_rec* d_recs1,
                                 uint8_t* d_seq2, uint8_t* d_qual2, uint16_t* d_len2, fp_fastq_rec* d_recs2,
                                 int64_t capacity, fp_fastq_info* info);
int  fp_fastq_encode_interleaved(fp_ctx* ctx, const uint8_t* d_text1, const fp_fastq_rec* d_recs1, const uint8_t* d_text2, const fp_fastq_rec* d_recs2,
                                 const fp_read_result* d_res1, const fp_read_result* d_res2,
                                 const uint8_t* d_seq1, const uint8_t* d_qual1, const uint8_t* d_seq2, const uint8_t* d_qual2,
                                 int64_t n, uint8_t* d_out, int64_t out_cap, int64_t* out_bytes);
int  fp_fastq_set_interleaved(fp_ctx* ctx, int32_t in, int32_t out);

/* ---------------- duplication bloom filter (SURVEY.md 8(f) rank 2; src/duplicate.cpp) ----------------
 * fp_dup_check replaces Duplicate::checkRead / checkPair (src/duplicate.cpp:126-154) for a batch in DEVICE memory: d_is_dup[i]
 * (nullable) = what the reference returns for unit i when units are fed in index order, batch after batch -- deterministic, not
 * the scheduling-dependent answer plain atomicOr would give (DESIGN.md).  The bit arrays live in the ctx (1 GiB at accuracy
 * level 1, --dup_accuracy_level src/main.cpp) and are allocated by the first call; later calls must use the same level.
 * fp_dup_totals: Duplicate::mTotalReads / mDupReads (getDupRate = dups / total).  Enqueued on `stream` (NULL = the ctx's).
 * Call it BEFORE fp_process_* on the same batch: the reference hashes the reads as they were read (checkPair comes before
 * any trimming or correction, src/peprocessor.cpp:397-401), and fp_process_pe corrects bases in place. */
int  fp_dup_check(fp_ctx* ctx, const fp_batch* b, int32_t accuracy_level, uint8_t* d_is_dup, void* stream);
int  fp_dup_totals(fp_ctx* ctx, int64_t* total, int64_t* dups);
int  fp_dup_reset(fp_ctx* ctx);
/* --dedup (src/options.h duplicate.dedup): `d_is_dup` = DEVICE flags of the batch the next fp_process_se / _pe call works on (as fp_dup_check
 * wrote them); flagged units keep their verdict counters but are left out of the post-filter stats and marked FP_F_DUPLICATE, which
 * fp_fastq_encode skips.  NULL switches it off.  The pointer stays set until it is changed: d_is_dup[i] belongs to unit i of the LAUNCH, so
 * a caller that splits a stream over several launches sets it before each one to that launch's first unit, and clears it when done.
 * In merging mode a merged read is counted and written whatever its flag says (src/peprocessor.cpp:528-534); only pairs that did not
 * merge consult it (:547, :553, :575).  The host entry points (fp_process_*_host, _host_packed, _host_patches, fp_fastq_process_host)
 * split their input into chunks and rounds of their own, so one flag array cannot follow them: while a pointer is set they return
 * FP_E_INVAL and touch nothing.  fp_fastq_set_dedup: the text path (fp_fastq_process_host, fp_fastq_process_host_merge) runs the duplicate filter at
 * `accuracy_level` on every round's decoded rows before the chain (0 = off) and drops duplicates from the output when `dedup` is set. */
int  fp_set_dup_flags(fp_ctx* ctx, const uint8_t* d_is_dup);
int  fp_fastq_set_dedup(fp_ctx* ctx, int32_t accuracy_level, int32_t dedup);

/* Host-side pre-scan (control plane, once per input, like the reference's Evaluator): the over-representation candidate list
 * Evaluator::computeOverRepSeq (src/evaluator.cpp:78-169) derives from the first 1.51 M bases of one input, here given as rows
 * in HOST memory.  Writes the sequences NUL-separated in the reference's map order; *n_out = how many, *bytes_out = bytes needed
 * (FP_E_TOOLARGE if out_cap is smaller).  seqlen = Options::seqLen1/2.  The result feeds fp_params.overrep_seqs1/2. */
int  fp_host_overrep_candidates(const uint8_t* seq, const uint16_t* len, int64_t n, int32_t stride, int32_t seqlen,
                                char* out, int64_t out_cap, int32_t* n_out, int64_t* bytes_out);

/* ---------------- gzip / BGZF either side of the text path (SURVEY.md 8(f) rank 4; host code on zlib) ----------------
 * fp_gz_inflate: a whole compressed buffer -> text; BGZF (src/bgzf.h:165-195) block-parallel on `threads` host threads, other gzip streams
 * member after member (src/fastqreader.cpp:88-209).  *n_out = decompressed size (FP_E_TOOLARGE if cap is smaller, BGZF only knows it upfront).
 * fp_gz_deflate: text -> concatenated gzip members of member_bytes input bytes each, compressed in parallel -- one member per output pack
 * is what the reference's writer threads produce (src/writerthread.cpp:118-168).  fp_gz_open / _read / _close: streaming reader (plain
 * files pass through) for callers that feed fp_fastq_process_host chunk by chunk.                                                  */
int     fp_gz_is_bgzf(const uint8_t* in, int64_t n);
int     fp_gz_inflate(const uint8_t* in, int64_t n_in, uint8_t* out, int64_t cap, int64_t* n_out, int threads);
int64_t fp_gz_deflate_bound(int64_t n_in, int64_t member_bytes);
int     fp_gz_deflate(const uint8_t* in, int64_t n_in, uint8_t* out, int64_t cap, int64_t* n_out, int64_t member_bytes, int level, int threads);
void*   fp_gz_open(const char* path);
int64_t fp_gz_read(void* h, uint8_t* buf, int64_t cap);
void    fp_gz_close(void* h);

/* Pinned host memory helpers for the staging shim. */
int  fp_host_alloc(void** p, size_t bytes);
int  fp_host_free(void* p);

/* Synthetic input generator (SURVEY.md 8(d)): fills DEVICE rows for reads/pairs
 * [first_index, first_index + b->n) of the stream identified by (seed, profile).  The same generator
 * compiled for the host (fastp_b200/csrc/synth.h via oracle/synth_host.c) regenerates any batch for the CPU oracle.
 * profile: 0 = ref-style (scripts/bench_e2e.sh:41-86), 1 = enriched fragment model.            */
int  fp_synth_fill(fp_ctx* ctx, const fp_batch* b, int64_t first_index, uint64_t seed,
                   int32_t profile, int32_t read_len, void* stream);

/* Timing hook: average duration in ms of the hot kernel launches recorded with CUDA events on the
 * launching stream since the last reset; returns number of launches through *n. */
int  fp_kernel_time_ms(fp_ctx* ctx, double* total_ms, int64_t* n_launches, int reset);

int  fp_version(void);

#ifdef __cplusplus
}
#endif
#endif /* FASTP_B200_H */
