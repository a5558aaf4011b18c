/*
 * fastp_oracle_merge.h -- CPU oracle of the merging-mode output streams of the text path.  TEST INFRASTRUCTURE ONLY
 * (see fastp_oracle_merge.c); built into oracle/libfastp_oracle_merge.so.
 */
#ifndef FASTP_ORACLE_MERGE_H
#define FASTP_ORACLE_MERGE_H
#include "fastp_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
/* Merging mode: one of the three output streams (`which` = FP_FQ_OUT_MERGED / _R1 / _R2) of src/peprocessor.cpp:519-622, merged reads built
 * as OverlapAnalysis::merge does (src/overlapanalysis.cpp:148-179).  Same arrays as fp_fastq_encode_merge, HOST pointers; returns the
 * size of the whole stream and writes the records that fit under out_cap. */
int64_t fp_oracle_fastq_encode_merge(int which, int include_unmerged, const uint8_t* text1, const fp_fastq_rec* recs1, const uint8_t* text2, const fp_fastq_rec* recs2,
                                     const fp_read_result* res1, const fp_read_result* res2, const fp_ov_result* ov,
                                     const uint8_t* seq1, const uint8_t* qual1, const uint8_t* seq2, const uint8_t* qual2,
                                     int stride, int64_t n, uint8_t* out, int64_t out_cap);
/* the complement a merged read's second half is written with (scalarReverseComplement, src/simd.cpp:296-308) */
uint8_t fp_oracle_merge_complement(uint8_t b);

#ifdef __cplusplus
}
#endif
#endif
