/*
 * fastp_oracle_index.h -- CPU oracle of the index filter (--filter_by_index1 / --filter_by_index2) of the text path.  TEST INFRASTRUCTURE
 * ONLY (see fastp_oracle_index.c); built into oracle/libfastp_oracle_index.so on top of libfastp_oracle.so.
 */
#ifndef FASTP_ORACLE_INDEX_H
#define FASTP_ORACLE_INDEX_H
#include "fastp_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
/* Read::firstIndex (first = 1) / Read::lastIndex (first = 0) of a name line of `len` bytes ('@' included): *start = where the index
 * begins; returns its length (0 for "") */
int64_t fp_oracle_index_of(const uint8_t* name, int64_t len, int first, int64_t* start);
/* Filter::match: whether any of the n barcodes of `list` (NUL-separated, one after the other) is within `threshold` differences of the
 * index over the shorter of the two */
int fp_oracle_index_match(const char* list, int64_t n, const uint8_t* index, int64_t len, int threshold);
/* Options::makeListFromFileByLine over a file's bytes: the barcodes NUL-separated into out (out_cap bytes; *out_bytes = bytes needed);
 * returns how many, or -1 where the reference stops with "each line should be one barcode, which can only contain A/T/C/G". */
int64_t fp_oracle_index_load(const uint8_t* data, int64_t nbytes, char* out, int64_t out_cap, int64_t* out_bytes);
/* Filter::filterByIndex for the records of a batch: flags[i] = 1 when unit i is removed.  text2 / recs2 NULL: single-end (list 1 against
 * firstIndex); else list 1 against read 1's firstIndex, then list 2 against read 2's lastIndex. */
void fp_oracle_index_flags(const uint8_t* text1, const fp_fastq_rec* recs1, const uint8_t* text2, const fp_fastq_rec* recs2, int64_t n,
                           const char* list1, int64_t n1, const char* list2, int64_t n2, int threshold, uint8_t* flags);
/* fp_oracle_process_dedup with the index filter: a unit with ix_flags[i] set goes through the pre-filter Stats (over-representation
 * sampling included) and nothing else: its records are the index-filtered record of fp_set_index_flags, its overlap record is zero and its
 * rows are left as they are (src/seprocessor.cpp:209-224, src/peprocessor.cpp:392-410).  is_dup nullable, as for fp_oracle_process_dedup.
 * Returns 0 or fp_oracle_process's error. */
int fp_oracle_process_index(const fp_params* p, const fp_counter_layout* L, const fp_batch* b, const uint8_t* is_dup, const uint8_t* ix_flags,
                            fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* counters);

#ifdef __cplusplus
}
#endif
#endif
