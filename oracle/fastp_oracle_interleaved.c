/*
 * fastp_oracle_interleaved.c -- plain-C restatement of reading and writing interleaved pairs: FastqReaderPair::read with interleaved = true
 * (src/fastqreader.cpp:452-460; the pair stream ends at the first NULL of either mate, ReadPair::eof src/read.cpp:203-205) over the
 * sequential record reader of fastp_oracle.c, and the --stdout stream of a paired run (src/peprocessor.cpp:579-581, singleOutput: read 1
 * then read 2 of every pair that out1 / out2 would get).  TEST INFRASTRUCTURE: the device's fp_fastq_decode_interleaved /
 * fp_fastq_encode_interleaved are compared with it, and tests/test_oracle_fastq_interleaved.py pins it to the reference's own
 * FastqReaderPair and to the unmodified reference CLI.  Links libfastp_oracle.so; never linked into the product.
 */
#include <stdlib.h>
#include <string.h>
#include "fastp_oracle.h"
#include "fastp_oracle_interleaved.h"

int fp_oracle_fastq_decode_interleaved(const uint8_t* text, int64_t nbytes, int final_chunk, int phred64, int stride,
                                       uint8_t* seq1, uint8_t* qual1, uint16_t* len1, fp_fastq_rec* recs1,
                                       uint8_t* seq2, uint8_t* qual2, uint16_t* len2, fp_fastq_rec* recs2,
                                       int64_t capacity, fp_fastq_info* info) {
    /* the records one by one, up to 2 * capacity of them */
    const int64_t cap = 2 * capacity;
    uint8_t* seq = (uint8_t*)calloc((size_t)(cap > 0 ? cap : 1), (size_t)stride);
    uint8_t* qual = (uint8_t*)calloc((size_t)(cap > 0 ? cap : 1), (size_t)stride);
    uint16_t* len = (uint16_t*)calloc((size_t)(cap > 0 ? cap : 1), sizeof(uint16_t));
    fp_fastq_rec* recs = (fp_fastq_rec*)calloc((size_t)(cap > 0 ? cap : 1), sizeof(fp_fastq_rec));
    int rc = -1;
    if (!seq || !qual || !len || !recs) goto done;
    fp_fastq_info one;
    if ((rc = fp_oracle_fastq_decode(text, nbytes, final_chunk, phred64, stride, seq, qual, len, cap, recs, &one))) goto done;
    *info = one;
    int64_t nrec = one.n_records;                             /* records before the first bad one, at most 2 * capacity */
    if (one.error == FP_FQ_OK && !one.more && (nrec & 1)) {   /* a lone mate 1 */
        if (final_chunk) info->consumed = nbytes;             /* its mate never comes: dropped, and the rest of the text with it */
        else info->consumed = recs[nrec - 1].name_off;        /* read again with its mate */
    }
    /* a bad record (mate 1 or 2) ends the pair stream before its pair: nrec records kept, nrec >> 1 pairs */
    info->n_records = nrec >> 1;
    for (int64_t r = 0; r < 2 * (nrec >> 1); r++) {
        const int64_t row = r >> 1;
        uint8_t* s = (r & 1) ? seq2 : seq1; uint8_t* q = (r & 1) ? qual2 : qual1;
        memcpy(s + (size_t)row * stride, seq + (size_t)r * stride, (size_t)stride);
        memcpy(q + (size_t)row * stride, qual + (size_t)r * stride, (size_t)stride);
        ((r & 1) ? len2 : len1)[row] = len[r];
        ((r & 1) ? recs2 : recs1)[row] = recs[r];
    }
done:
    free(seq); free(qual); free(len); free(recs);
    return rc;
}

int64_t fp_oracle_fastq_encode_interleaved(const uint8_t* text1, const fp_fastq_rec* recs1, const uint8_t* text2, const fp_fastq_rec* recs2,
                                           const fp_read_result* res1, const fp_read_result* res2,
                                           const uint8_t* seq1, const uint8_t* qual1, const uint8_t* seq2, const uint8_t* qual2,
                                           int stride, int64_t n, uint8_t* out, int64_t out_cap) {
    int64_t o = 0;
    for (int64_t i = 0; i < n; i++) {
        const size_t row = (size_t)i * stride;
        for (int side = 0; side < 2; side++) {
            const int64_t room = out && o < out_cap ? out_cap - o : 0;
            o += fp_oracle_fastq_encode(side ? text2 : text1, (side ? recs2 : recs1) + i, (side ? res2 : res1) + i, (side ? seq2 : seq1) + row,
                                        (side ? qual2 : qual1) + row, stride, 1, room > 0 ? out + o : NULL, room);
        }
    }
    return o;
}
