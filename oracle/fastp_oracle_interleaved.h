/*
 * fastp_oracle_interleaved.h -- CPU oracle of interleaved FASTQ on the text path (--interleaved_in, --stdout for pairs).  TEST
 * INFRASTRUCTURE ONLY (see fastp_oracle_interleaved.c); built into oracle/libfastp_oracle_interleaved.so.
 */
#ifndef FASTP_ORACLE_INTERLEAVED_H
#define FASTP_ORACLE_INTERLEAVED_H
#include "fastp_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
/* fp_fastq_decode_interleaved on HOST pointers: record r of the chunk goes to side (r & 1), row (r >> 1); capacity and info->n_records
 * count pairs, info->error_record counts records of the text. */
int fp_oracle_fastq_decode_interleaved(const uint8_t* text, int64_t nbytes, int final_chunk, int phred64, int stride,
                                       uint8_t* seq1, uint8_t* qual1, uint16_t* len1, fp_fastq_rec* recs1,
                                       uint8_t* seq2, uint8_t* qual2, uint16_t* len2, fp_fastq_rec* recs2,
                                       int64_t capacity, fp_fastq_info* info);
/* fp_fastq_encode_interleaved on HOST pointers: per pair, read 1's record as fp_oracle_fastq_encode writes it, then read 2's.  Returns the
 * size of the whole stream and writes the records that fit under out_cap. */
int64_t fp_oracle_fastq_encode_interleaved(const uint8_t* text1, const fp_fastq_rec* recs1, const uint8_t* text2, const fp_fastq_rec* recs2,
                                           const fp_read_result* res1, const fp_read_result* res2,
                                           const uint8_t* seq1, const uint8_t* qual1, const uint8_t* seq2, const uint8_t* qual2,
                                           int stride, int64_t n, uint8_t* out, int64_t out_cap);
#ifdef __cplusplus
}
#endif
#endif
