/*
 * fastp_oracle_overlapped.h -- CPU oracle of the --overlapped_out stream of the text path.  TEST INFRASTRUCTURE ONLY
 * (see fastp_oracle_overlapped.c); built into oracle/libfastp_oracle_overlapped.so on top of libfastp_oracle.so.
 */
#ifndef FASTP_ORACLE_OVERLAPPED_H
#define FASTP_ORACLE_OVERLAPPED_H
#include "fastp_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
/* The analysis src/peprocessor.cpp:488-495 runs for --overlapped_out, for every pair of a HOST batch (paired params only): ovx[i] =
 * OverlapAnalysis::analyze(r1, r2, overlapDiffLimit, overlapRequire, 0) on the two reads as the adapter trimmers left them, with read 1's
 * length then, or all zero when trimAndCut dropped a read.  The rows are changed in place by base correction, as fp_oracle_process changes them; L is the
 * layout of the run (scratch counters).  Returns 0 or fp_oracle_process's error. */
int fp_oracle_overlapped_analyze(const fp_params* p, const fp_counter_layout* L, const fp_batch* b, fp_overlapped_result* ovx);
/* The --overlapped_out text of a batch: for every unit whose two reads trimAndCut kept (FP_F_DROPPED of res1 / res2) and whose ovx
 * overlapped, read 1's name line, std::string(r1.substr(max(0, offset)), overlap_len) -- read 1 AFTER the overlap, row bytes
 * [front + max(0, offset) + overlap_len, front + r1_len) of seq1 / qual1 (rows of `stride` bytes) -- and read 1's strand line
 * (Read::appendToString, src/read.cpp:119-134).  Returns the size of the whole stream and writes the records that fit under out_cap. */
int64_t fp_oracle_fastq_encode_overlapped(const uint8_t* text1, const fp_fastq_rec* recs1, const fp_read_result* res1, const fp_read_result* res2,
                                          const fp_overlapped_result* ovx, const uint8_t* seq1, const uint8_t* qual1, int stride, int64_t n,
                                          uint8_t* out, int64_t out_cap);

#ifdef __cplusplus
}
#endif
#endif
