/*
 * fastp_oracle_overlapped.c -- plain-C restatement of what PairEndProcessor::processPairEnd (src/peprocessor.cpp:488-495) writes to
 * --overlapped_out.  TEST INFRASTRUCTURE: the device chain's analysis (fp_set_overlapped_sink) and encoder (fp_fastq_encode_overlapped)
 * are compared with it, and tests/test_oracle_fastq_overlapped.py pins it to the unmodified reference CLI's file.  Written from the
 * reference's behaviour; never linked into the product.
 */
#include <stdlib.h>
#include <string.h>
#include "fastp_oracle.h"
#include "fastp_oracle_overlapped.h"

/* The analysis sees r1 / r2 after trimAndCut, polyG, base correction and the adapter trimmers (:425-485) and before polyX and the
   max_len clip (:506-516).  Neither of those two changes anything the steps before them see, and both only shorten a read from its 3'
   end, so the windows the analysis sees are the records of the same run with both of them switched off. */
int fp_oracle_overlapped_analyze(const fp_params* p, const fp_counter_layout* L, const fp_batch* b, fp_overlapped_result* ovx) {
    const int64_t n = b->n;
    fp_params q = *p;
    q.polyx_enabled = 0; q.max_len1 = 0; q.max_len2 = 0;
    fp_read_result* w = (fp_read_result*)calloc((size_t)(2 * n + 1), sizeof(fp_read_result));
    fp_ov_result* ov = (fp_ov_result*)calloc((size_t)(n + 1), sizeof(fp_ov_result));
    int64_t* counters = (int64_t*)calloc((size_t)L->total + 1, sizeof(int64_t));
    int rc = (w && ov && counters) ? fp_oracle_process(&q, L, b, w, w + n, ov, counters) : -1;
    for (int64_t i = 0; rc == 0 && i < n; i++) {
        const fp_read_result *a = &w[i], *c = &w[n + i];
        memset(&ovx[i], 0, sizeof(ovx[i]));
        if ((a->flags | c->flags) & FP_F_DROPPED) continue;                                           /* r1 && r2 (:488) */
        const fp_ov_result o = fp_oracle_analyze(b->seq1 + (size_t)i * b->stride + a->front, a->len, b->seq2 + (size_t)i * b->stride + c->front,
                                                 c->len, p->overlap_diff_limit, p->overlap_require, 0.0);
        ovx[i].overlapped = o.overlapped; ovx[i].offset = o.offset; ovx[i].overlap_len = o.overlap_len; ovx[i].r1_len = (uint16_t)a->len;
    }
    free(w); free(ov); free(counters);
    return rc;
}

int64_t fp_oracle_fastq_encode_overlapped(const uint8_t* text1, const fp_fastq_rec* recs1, const fp_read_result* res1, const fp_read_result* res2,
                                          const fp_overlapped_result* ovx, const uint8_t* seq1, const uint8_t* qual1, int stride, int64_t n,
                                          uint8_t* out, int64_t out_cap) {
    int64_t o = 0;
    for (int64_t i = 0; i < n; i++) {
        if (!ovx[i].overlapped || ((res1[i].flags | res2[i].flags) & FP_F_DROPPED)) continue;
        /* std::string(r1.substr(max(0, offset)), overlap_len): overlap_len is the constructor's start position */
        const int64_t skip = (ovx[i].offset > 0 ? ovx[i].offset : 0) + ovx[i].overlap_len;
        const int64_t from = (int64_t)i * stride + res1[i].front + skip, len = ovx[i].r1_len > skip ? ovx[i].r1_len - skip : 0;
        const fp_fastq_rec* rc = &recs1[i];
        const int64_t nl = rc->name_len, sl = rc->strand_len, need = nl + sl + 2 * len + 4;
        if (o + need <= out_cap) {
            uint8_t* d = out + o;
            memcpy(d, text1 + rc->name_off, (size_t)nl); d += nl; *d++ = '\n';
            memcpy(d, seq1 + from, (size_t)len); d += len; *d++ = '\n';
            memcpy(d, text1 + rc->strand_off, (size_t)sl); d += sl; *d++ = '\n';
            memcpy(d, qual1 + from, (size_t)len); d += len; *d++ = '\n';
        }
        o += need;
    }
    return o;
}
