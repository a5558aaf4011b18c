/*
 * fastp_oracle.h -- CPU oracle of the per-read hot path.  TEST INFRASTRUCTURE ONLY (see fastp_oracle.c).
 */
#ifndef FASTP_ORACLE_H
#define FASTP_ORACLE_H
#include "fastp_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
/* Runs processSingleEnd / processPairEnd semantics over a HOST batch; per-read records to out1/out2
 * (out2, ov may be NULL for SE / if unwanted); counters are ADDED into counters[L->total].
 * seq/qual rows are modified in place by base correction. */
int fp_oracle_process(const fp_params* p, const fp_counter_layout* L, const fp_batch* b,
                      fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* counters);
/* The same with --dedup: is_dup[b->n] (nullable = fp_oracle_process) are the duplicate filter's answers with duplicate.dedup set,
 * i.e. dedupOut of src/seprocessor.cpp:280 and src/peprocessor.cpp:397-401.  A flagged unit keeps its FilterResult counters, gets
 * FP_F_DUPLICATE and is left out of the post-filter Stats (:575) -- except in merging mode, where a MERGED read is counted whatever
 * the flag says (:528-534) and only the --include_unmerged branch consults it (:547, :553). */
int fp_oracle_process_dedup(const fp_params* p, const fp_counter_layout* L, const fp_batch* b, const uint8_t* is_dup,
                            fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* counters);

/* single-operator entry points for known-answer tests */
int fp_oracle_trim_and_cut(const fp_params* p, uint8_t* seq, uint8_t* qual, int len, int front, int tail, int* frontOut, int* lenOut);
int fp_oracle_trim_polyg(uint8_t* seq, int len, int minLen);
int fp_oracle_trim_polyx(uint8_t* seq, int len, int minLen, int* poly, int* plen);
int fp_oracle_trim_by_sequence(uint8_t* seq, int len, const char* adapter, int* trimmed);
fp_ov_result fp_oracle_analyze(uint8_t* seq1, int len1, uint8_t* seq2, int len2, int diffLimit, int overlapRequire, double diffPercentLimit);
int fp_oracle_pass_filter(const fp_params* p, uint8_t* seq, uint8_t* qual, int len);
int fp_oracle_match_with_one_insertion(const uint8_t* insData, const uint8_t* normalData, int cmplen, int diffLimit);

/* FASTQ text <-> rows: FastqReader::getLine / read (src/fastqreader.cpp:240-368) and Read::appendToString (src/read.cpp:119-134)
 * restated over an in-memory chunk; same arguments and results as fp_fastq_decode / fp_fastq_encode (records with FP_F_DUPLICATE are
 * not written), HOST pointers. */
int fp_oracle_fastq_decode(const uint8_t* text, int64_t nbytes, int final_chunk, int phred64, int stride,
                           uint8_t* seq, uint8_t* qual, uint16_t* len, int64_t capacity, fp_fastq_rec* recs, fp_fastq_info* info);
int64_t fp_oracle_fastq_encode(const uint8_t* text, const fp_fastq_rec* recs, const fp_read_result* res, const uint8_t* seq, const uint8_t* qual,
                               int stride, int64_t n, uint8_t* out, int64_t out_cap);

/* Duplication bloom filter (SURVEY 8f rank 2; src/duplicate.cpp) -- the sequential form fp_dup_check is compared with.
 * is_dup[i] = what Duplicate::checkRead / checkPair returns for unit i when the units are fed in index order. */
typedef struct fp_oracle_dup fp_oracle_dup;
fp_oracle_dup* fp_oracle_dup_create(int accuracy_level);
void fp_oracle_dup_destroy(fp_oracle_dup* d);
void fp_oracle_dup_check(fp_oracle_dup* d, const fp_batch* b, int paired, uint8_t* is_dup);
void fp_oracle_dup_totals(const fp_oracle_dup* d, int64_t* total, int64_t* dups);
#ifdef __cplusplus
}
#endif
#endif
