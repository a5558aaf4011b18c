/*
 * fastp_oracle_outs.h -- CPU oracle of the --unpaired1 / --unpaired2 / --failed_out streams of the text path.  TEST INFRASTRUCTURE ONLY
 * (see fastp_oracle_outs.c); built into oracle/libfastp_oracle_outs.so.
 */
#ifndef FASTP_ORACLE_OUTS_H
#define FASTP_ORACLE_OUTS_H
#include "fastp_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
/* One of the streams `which` = FP_FQ_OUT_UNPAIRED1 / _UNPAIRED2 / _FAILED of src/seprocessor.cpp:280-290 (paired = 0) or
 * src/peprocessor.cpp:575-620 (paired = 1), with the unpaired writers `writers` (FP_FQ_W_*) that exist; merging = the run merges pairs
 * (then only pairs that took neither merging branch write here).  Same arrays as fp_fastq_encode_rejects, HOST pointers; returns the size
 * of the whole stream and writes the records that fit under out_cap. */
int64_t fp_oracle_fastq_encode_rejects(int which, int writers, int paired, int merging, int include_unmerged,
                                       const uint8_t* text1, const fp_fastq_rec* recs1, const uint8_t* text2, const fp_fastq_rec* recs2,
                                       const fp_read_result* res1, const fp_read_result* res2,
                                       const uint8_t* seq1, const uint8_t* qual1, const uint16_t* len1,
                                       const uint8_t* seq2, const uint8_t* qual2, const uint16_t* len2,
                                       int stride, int64_t n, uint8_t* out, int64_t out_cap);

#ifdef __cplusplus
}
#endif
#endif
