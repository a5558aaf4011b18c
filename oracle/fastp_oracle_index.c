/*
 * fastp_oracle_index.c -- plain-C restatement of the index filter: Options::makeListFromFileByLine (src/options.cpp:484-510),
 * Read::firstIndex / lastIndex (src/read.cpp:75-100), Filter::filterByIndex / match (src/filter.cpp:209-243) and where the per-read loops
 * drop a filtered unit (src/seprocessor.cpp:209-224, src/peprocessor.cpp:392-410).  TEST INFRASTRUCTURE: the device matcher
 * (fp_fastq_index_flags) and the chain's index flags (fp_set_index_flags) are compared with it, and tests/test_oracle_fastq_index.py pins
 * it to the unmodified reference CLI.  Written from the reference's behaviour; never linked into the product.
 */
#include <stdlib.h>
#include <string.h>
#include "fastp_oracle.h"
#include "fastp_oracle_index.h"

int64_t fp_oracle_index_of(const uint8_t* name, int64_t len, int first, int64_t* start) {
    *start = 0;
    if (len < 5) return 0;
    int64_t end = len;                                    /* firstIndex: the last '+' met, walking down, ends the index before it */
    for (int64_t i = len - 3; i >= 0; i--) {
        if (first && name[i] == '+') end = i - 1;
        if (name[i] == ':' || (!first && name[i] == '+')) {
            /* substr(i + 1, count): count = end - i (firstIndex) or len - i (lastIndex), cut at the end of the name */
            const int64_t count = first ? end - i : len - i;
            *start = i + 1;
            return count < len - (i + 1) ? count : len - (i + 1);
        }
    }
    return 0;
}

int fp_oracle_index_match(const char* list, int64_t n, const uint8_t* index, int64_t len, int threshold) {
    for (int64_t k = 0; k < n; k++) {
        const int64_t blen = (int64_t)strlen(list);
        int diff = 0;
        for (int64_t s = 0; s < blen && s < len; s++) {
            if ((uint8_t)list[s] != index[s]) {
                diff++;
                if (diff > threshold) break;
            }
        }
        if (diff <= threshold) return 1;
        list += blen + 1;
    }
    return 0;
}

/* istream::getline(line, 1000) over the bytes: up to 999 characters or the '\n' (taken, not kept).  Returns 1 and the line, or 0 when the
   stream fails: nothing left to read, or 999 characters with more of the line to come. */
static int getline_1000(const uint8_t* d, int64_t n, int64_t* pos, char* line) {
    int64_t i = *pos, k = 0;
    if (i >= n) return 0;
    while (k + 1 < 1000 && i < n && d[i] != '\n') line[k++] = (char)d[i++];
    line[k] = '\0';
    if (i < n && d[i] == '\n') i++;
    else if (i < n) return 0;                             /* line longer than the buffer: failbit */
    *pos = i;
    return 1;
}

int64_t fp_oracle_index_load(const uint8_t* data, int64_t nbytes, char* out, int64_t out_cap, int64_t* out_bytes) {
    char line[1000];
    int64_t pos = 0, count = 0, o = 0;
    while (getline_1000(data, nbytes, &pos, line)) {
        const size_t got = strlen(line);
        if (got >= 2 && (line[got - 1] == '\n' || line[got - 1] == '\r')) {
            line[got - 1] = '\0';
            if (line[got - 2] == '\r') line[got - 2] = '\0';
        }
        const size_t bl = strlen(line);
        for (size_t t = 0; t < bl; t++)
            if (line[t] != 'A' && line[t] != 'T' && line[t] != 'C' && line[t] != 'G') return -1;
        if (o + (int64_t)bl + 1 <= out_cap) memcpy(out + o, line, bl + 1);
        o += (int64_t)bl + 1;
        count++;
    }
    *out_bytes = o;
    return count;
}

void fp_oracle_index_flags(const uint8_t* text1, const fp_fastq_rec* recs1, const uint8_t* text2, const fp_fastq_rec* recs2, int64_t n,
                           const char* list1, int64_t n1, const char* list2, int64_t n2, int threshold, uint8_t* flags) {
    for (int64_t i = 0; i < n; i++) {
        int64_t s, len;
        const uint8_t* name1 = text1 + recs1[i].name_off;
        len = fp_oracle_index_of(name1, recs1[i].name_len & 0x0FFFFFFFu, 1, &s);
        int f = fp_oracle_index_match(list1, n1, name1 + s, len, threshold);
        if (!f && text2) {
            const uint8_t* name2 = text2 + recs2[i].name_off;
            len = fp_oracle_index_of(name2, recs2[i].name_len & 0x0FFFFFFFu, 0, &s);
            f = fp_oracle_index_match(list2, n2, name2 + s, len, threshold);
        }
        flags[i] = (uint8_t)f;
    }
}

static fp_read_result filtered_record(void) {
    fp_read_result r;
    memset(&r, 0, sizeof(r));
    r.verdict = r.pair_verdict = FP_FAIL_LENGTH; r.flags = FP_F_DROPPED; r.polyx_base = 255; r.flags2 = FP_F2_INDEX_FILTERED;
    return r;
}

static uint8_t* dup_bytes(const void* src, size_t n) {
    uint8_t* d = (uint8_t*)malloc(n ? n : 1);
    if (d && n) memcpy(d, src, n);
    return d;
}

/* The pre-filter Stats (blocks FP_STATS_PRE1 / PRE2 and their over-representation regions) see every unit in input order, and the rest of
   the counters only the units that stay.  So: the whole batch, on copies of its rows, gives the pre-filter blocks; the batch of the units
   that stay, started from the same counters, gives everything else, their records and their corrected rows. */
int fp_oracle_process_index(const fp_params* p, const fp_counter_layout* L, const fp_batch* b, const uint8_t* is_dup, const uint8_t* ix_flags,
                            fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* counters) {
    const int64_t n = b->n, S = b->stride;
    const int paired = p->paired != 0;
    const size_t rows = (size_t)n * (size_t)S;
    int64_t k = 0;
    for (int64_t i = 0; i < n; i++) k += ix_flags[i] == 0;
    int64_t* cpre = (int64_t*)dup_bytes(counters, (size_t)L->total * 8);
    fp_read_result* w = (fp_read_result*)calloc((size_t)(2 * n + 2), sizeof(fp_read_result));
    fp_ov_result* wov = (fp_ov_result*)calloc((size_t)(n + 1), sizeof(fp_ov_result));
    fp_batch all = *b;
    all.seq1 = dup_bytes(b->seq1, rows); all.qual1 = dup_bytes(b->qual1, rows);
    if (paired) { all.seq2 = dup_bytes(b->seq2, rows); all.qual2 = dup_bytes(b->qual2, rows); }
    int rc = (cpre && w && wov && all.seq1 && all.qual1 && (!paired || (all.seq2 && all.qual2))) ? 0 : -1;
    if (rc == 0) rc = fp_oracle_process_dedup(p, L, &all, is_dup, w, paired ? w + n : NULL, paired ? wov : NULL, cpre);
    /* the units that stay, packed */
    fp_batch kb = *b;
    kb.n = k;
    kb.seq1 = (uint8_t*)malloc((size_t)k * S + 1); kb.qual1 = (uint8_t*)malloc((size_t)k * S + 1); kb.len1 = (uint16_t*)malloc((size_t)k * 2 + 2);
    if (paired) { kb.seq2 = (uint8_t*)malloc((size_t)k * S + 1); kb.qual2 = (uint8_t*)malloc((size_t)k * S + 1); kb.len2 = (uint16_t*)malloc((size_t)k * 2 + 2); }
    uint8_t* kdup = is_dup ? (uint8_t*)malloc((size_t)k + 1) : NULL;
    fp_read_result* k1 = (fp_read_result*)calloc((size_t)(k + 1), sizeof(fp_read_result));
    fp_read_result* k2 = (fp_read_result*)calloc((size_t)(k + 1), sizeof(fp_read_result));
    fp_ov_result* kov = (fp_ov_result*)calloc((size_t)(k + 1), sizeof(fp_ov_result));
    if (!kb.seq1 || !kb.qual1 || !kb.len1 || (paired && (!kb.seq2 || !kb.qual2 || !kb.len2)) || (is_dup && !kdup) || !k1 || !k2 || !kov) rc = -1;
    for (int64_t i = 0, j = 0; rc == 0 && i < n; i++) {
        if (ix_flags[i]) continue;
        memcpy(kb.seq1 + j * S, b->seq1 + i * S, (size_t)S); memcpy(kb.qual1 + j * S, b->qual1 + i * S, (size_t)S); kb.len1[j] = b->len1[i];
        if (paired) { memcpy(kb.seq2 + j * S, b->seq2 + i * S, (size_t)S); memcpy(kb.qual2 + j * S, b->qual2 + i * S, (size_t)S); kb.len2[j] = b->len2[i]; }
        if (kdup) kdup[j] = is_dup[i];
        j++;
    }
    if (rc == 0 && k > 0) rc = fp_oracle_process_dedup(p, L, &kb, kdup, k1, paired ? k2 : NULL, paired ? kov : NULL, counters);
    if (rc == 0) {
        const int pre[2] = {FP_STATS_PRE1, FP_STATS_PRE2};
        for (int t = 0; t < (paired ? 2 : 1); t++) {
            const int s = pre[t];
            memcpy(counters + s * L->stats_stride, cpre + s * L->stats_stride, (size_t)L->stats_stride * 8);
            const int64_t words = (int64_t)L->n_overrep[s >> 1] * (1 + L->overrep_len[s >> 1]);
            memcpy(counters + L->off_overrep[s], cpre + L->off_overrep[s], (size_t)words * 8);
        }
        for (int64_t i = 0, j = 0; i < n; i++) {
            if (ix_flags[i]) {
                out1[i] = filtered_record();
                if (paired) { out2[i] = filtered_record(); if (ov) memset(&ov[i], 0, sizeof(ov[i])); }
                continue;
            }
            out1[i] = k1[j];
            memcpy(b->seq1 + i * S, kb.seq1 + j * S, (size_t)S); memcpy(b->qual1 + i * S, kb.qual1 + j * S, (size_t)S);
            if (paired) {
                out2[i] = k2[j];
                if (ov) ov[i] = kov[j];
                memcpy(b->seq2 + i * S, kb.seq2 + j * S, (size_t)S); memcpy(b->qual2 + i * S, kb.qual2 + j * S, (size_t)S);
            }
            j++;
        }
    }
    free(cpre); free(w); free(wov);
    free(all.seq1); free(all.qual1); if (paired) { free(all.seq2); free(all.qual2); }
    free(kb.seq1); free(kb.qual1); free(kb.len1);
    if (paired) { free(kb.seq2); free(kb.qual2); free(kb.len2); }
    free(kdup); free(k1); free(k2); free(kov);
    return rc;
}
