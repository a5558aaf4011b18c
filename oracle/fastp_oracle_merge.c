/*
 * fastp_oracle_merge.c -- plain-C restatement of what PairEndProcessor::processPairEnd writes in merging mode
 * (src/peprocessor.cpp:519-622) and of OverlapAnalysis::merge (src/overlapanalysis.cpp:148-179), over the records the operator
 * chain produced.  TEST INFRASTRUCTURE: the device encoder (fp_fastq_encode_merge) is compared with it, and
 * tests/test_oracle_fastq_merge.py pins it to the unmodified reference CLI's files.  Written from the reference's behaviour;
 * never linked into the product.
 */
#include <string.h>
#include "fastp_oracle_merge.h"
#include <stdio.h>
/* scalarReverseComplement  src/simd.cpp:296-308, one base */
uint8_t fp_oracle_merge_complement(uint8_t b) {
    switch (b) {
        case 'A': case 'a': return 'T';
        case 'T': case 't': return 'A';
        case 'C': case 'c': return 'G';
        case 'G': case 'g': return 'C';
        default: return 'N';
    }
}

/* appends one record (Read::appendToString src/read.cpp:119-134) at *o if it fits; *o advances either way */
static void fq_append(uint8_t* out, int64_t out_cap, int64_t* o, const uint8_t* name, int64_t nl, const uint8_t* bases, const uint8_t* strand, int64_t sl,
                      const uint8_t* quals, int64_t len) {
    const int64_t need = nl + sl + 2 * len + 4;
    if (*o + need <= out_cap) {
        uint8_t* d = out + *o;
        memcpy(d, name, (size_t)nl); d += nl; *d++ = '\n';
        memcpy(d, bases, (size_t)len); d += len; *d++ = '\n';
        memcpy(d, strand, (size_t)sl); d += sl; *d++ = '\n';
        memcpy(d, quals, (size_t)len); d += len; *d++ = '\n';
    }
    *o += need;
}

int64_t fp_oracle_fastq_encode_merge(int which, int include_unmerged, const uint8_t* text1, const fp_fastq_rec* recs1, const uint8_t* text2, const fp_fastq_rec* recs2,
                                     const fp_read_result* res1, const fp_read_result* res2, const fp_ov_result* ov,
                                     const uint8_t* seq1, const uint8_t* qual1, const uint8_t* seq2, const uint8_t* qual2,
                                     int stride, int64_t n, uint8_t* out, int64_t out_cap) {
    int64_t o = 0;
    for (int64_t i = 0; i < n; i++) {
        const fp_read_result* a = res1 + i; const fp_read_result* b = res2 + i;
        const uint8_t* s1 = seq1 + (size_t)i * stride + a->front; const uint8_t* q1 = qual1 + (size_t)i * stride + a->front;
        const uint8_t* s2 = seq2 + (size_t)i * stride + b->front; const uint8_t* q2 = qual2 + (size_t)i * stride + b->front;
        if (a->flags & FP_F_MERGED) {                                           /* peprocessor.cpp:525-536: nothing of this pair reaches out1 / out2 */
            if (which != FP_FQ_OUT_MERGED || a->verdict != FP_PASS_FILTER) continue;    /* :529, dedupOut not consulted */
            int len1, len2;
            fp_merged_lens(ov + i, b->len, &len1, &len2);                     /* overlapanalysis.cpp:153-156 */
            uint8_t name[4096 + 64], strand[4096 + 64], bases[2 * FP_MAX_STRIDE], quals[2 * FP_MAX_STRIDE];
            char suffix[64];
            const int sufl = snprintf(suffix, sizeof(suffix), " merged_%d_%d", len1, len2);      /* :171 */
            int64_t nl = recs1[i].name_len, sl = recs1[i].strand_len;
            if (nl > 4096 || sl > 4096) return -1;                             /* longer lines than this checker holds */
            memcpy(name, text1 + recs1[i].name_off, (size_t)nl); memcpy(name + nl, suffix, (size_t)sufl); nl += sufl;
            memcpy(strand, text1 + recs1[i].strand_off, (size_t)sl);
            if (!(sl == 1 && strand[0] == '+')) { memcpy(strand + sl, suffix, (size_t)sufl); sl += sufl; }   /* :173-175 */
            memcpy(bases, s1, (size_t)len1); memcpy(quals, q1, (size_t)len1);  /* :159, :164 */
            for (int k = 0; k < len2; k++) {                                   /* :161, :166: reverseComplement(r2)[ol + k] = complement(r2[len2 - 1 - k]) */
                bases[len1 + k] = fp_oracle_merge_complement(s2[len2 - 1 - k]);
                quals[len1 + k] = q2[len2 - 1 - k];
            }
            fq_append(out, out_cap, &o, name, nl, bases, strand, sl, quals, len1 + len2);
        } else if (include_unmerged && !((a->flags | b->flags) & FP_F_DROPPED)) {      /* :521 r1 && r2, :537-556 */
            if (which != FP_FQ_OUT_MERGED) continue;
            if (a->verdict == FP_PASS_FILTER && !(a->flags & FP_F_DUPLICATE))   /* :547 */
                fq_append(out, out_cap, &o, text1 + recs1[i].name_off, recs1[i].name_len, s1, text1 + recs1[i].strand_off, recs1[i].strand_len, q1, a->len);
            if (b->verdict == FP_PASS_FILTER && !(b->flags & FP_F_DUPLICATE))   /* :553 */
                fq_append(out, out_cap, &o, text2 + recs2[i].name_off, recs2[i].name_len, s2, text2 + recs2[i].strand_off, recs2[i].strand_len, q2, b->len);
        } else {                                                                /* :563-585 */
            if (which == FP_FQ_OUT_MERGED || a->pair_verdict != FP_PASS_FILTER || (a->flags & FP_F_DUPLICATE)) continue;
            if (which == FP_FQ_OUT_R1)
                fq_append(out, out_cap, &o, text1 + recs1[i].name_off, recs1[i].name_len, s1, text1 + recs1[i].strand_off, recs1[i].strand_len, q1, a->len);
            else
                fq_append(out, out_cap, &o, text2 + recs2[i].name_off, recs2[i].name_len, s2, text2 + recs2[i].strand_off, recs2[i].strand_len, q2, b->len);
        }
    }
    return o;
}

