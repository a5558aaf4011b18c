/*
 * fastp_oracle_outs.c -- plain-C restatement of what SingleEndProcessor::processSingleEnd (src/seprocessor.cpp:280-290) and
 * PairEndProcessor::processPairEnd (src/peprocessor.cpp:575-620) write to --unpaired1, --unpaired2 and --failed_out, over the records
 * the operator chain produced.  TEST INFRASTRUCTURE: the device encoder (fp_fastq_encode_rejects) is compared with it, and
 * tests/test_oracle_fastq_outs.py pins it to the unmodified reference CLI's files.  Written from the reference's behaviour; never linked
 * into the product.
 */
#include <string.h>
#include "fastp_oracle_outs.h"

/* FAILED_TYPES src/common.h:56-65 */
static const char* const FAILED_TYPES[FP_FILTER_RESULT_TYPES] = {
    "passed", "", "", "",
    "failed_polyx_filter", "", "", "",
    "failed_bad_overlap", "", "", "",
    "failed_too_many_n_bases", "", "", "",
    "failed_too_short", "failed_too_long", "", "",
    "failed_quality_filter", "", "", "",
    "failed_low_complexity", "", "", "",
    "failed_adapter_dimer", "", "", ""};

/* one side of one unit as the reference holds it: r = the read after trimAndCut (NULL when dropped), or = the read as it was read,
   which trimAndCut and every later operator changed in place whenever they kept it (so or == r unless r == NULL) */
typedef struct {
    const uint8_t *text, *seq, *qual;
    const fp_fastq_rec* rec;
    const fp_read_result* res;
    int decoded_len;
} side_t;

/* Read::appendToString (tag == NULL, src/read.cpp:119-134) or Read::appendToStringWithTag (src/read.cpp:136-154) of `or`: the kept window,
   or the whole row for a dropped read; the record is written only if it fits, *o advances either way */
static void append_or(uint8_t* out, int64_t out_cap, int64_t* o, const side_t* s, const char* tag) {
    const int dropped = (s->res->flags & FP_F_DROPPED) != 0;
    const int64_t from = dropped ? 0 : s->res->front, len = dropped ? s->decoded_len : s->res->len;
    const int64_t nl = s->rec->name_len, sl = s->rec->strand_len, tl = tag ? (int64_t)strlen(tag) : 0;
    const int64_t need = nl + (tag ? 1 + tl : 0) + sl + 2 * len + 4;
    if (*o + need <= out_cap) {
        uint8_t* d = out + *o;
        memcpy(d, s->text + s->rec->name_off, (size_t)nl); d += nl;
        if (tag) { *d++ = ' '; memcpy(d, tag, (size_t)tl); d += tl; }
        *d++ = '\n';
        memcpy(d, s->seq + from, (size_t)len); d += len; *d++ = '\n';
        memcpy(d, s->text + s->rec->strand_off, (size_t)sl); d += sl; *d++ = '\n';
        memcpy(d, s->qual + from, (size_t)len); d += len; *d++ = '\n';
    }
    *o += need;
}

int64_t fp_oracle_fastq_encode_rejects(int which, int writers, int paired, int merging, int include_unmerged,
                                       const uint8_t* text1, const fp_fastq_rec* recs1, const uint8_t* text2, const fp_fastq_rec* recs2,
                                       const fp_read_result* res1, const fp_read_result* res2,
                                       const uint8_t* seq1, const uint8_t* qual1, const uint16_t* len1,
                                       const uint8_t* seq2, const uint8_t* qual2, const uint16_t* len2,
                                       int stride, int64_t n, uint8_t* out, int64_t out_cap) {
    const int unpairedLeft = (writers & FP_FQ_W_UNPAIRED1) != 0, unpairedRight = (writers & FP_FQ_W_UNPAIRED2) != 0;
    /* the strings the loop appends to (peprocessor.cpp:575-620); only the one asked for is built */
    const int toFailed = which == FP_FQ_OUT_FAILED, toUnpaired1 = which == FP_FQ_OUT_UNPAIRED1, toUnpaired2 = which == FP_FQ_OUT_UNPAIRED2;
    int64_t o = 0;
    for (int64_t i = 0; i < n; i++) {
        side_t or1 = {text1, seq1 + (size_t)i * stride, qual1 + (size_t)i * stride, recs1 + i, res1 + i, len1[i]};
        const int dedupOut = (res1[i].flags & FP_F_DUPLICATE) != 0;
        const int r1 = !(res1[i].flags & FP_F_DROPPED), result1 = res1[i].verdict;      /* verdict: passFilter after the dimer override */
        if (!paired) {                                                               /* seprocessor.cpp:280-290 */
            if (!dedupOut && !(r1 && result1 == FP_PASS_FILTER) && toFailed) append_or(out, out_cap, &o, &or1, FAILED_TYPES[result1]);
            continue;
        }
        side_t or2 = {text2, seq2 + (size_t)i * stride, qual2 + (size_t)i * stride, recs2 + i, res2 + i, len2[i]};
        const int r2 = !(res2[i].flags & FP_F_DROPPED), result2 = res2[i].verdict;
        if (merging && r1 && r2 && ((res1[i].flags & FP_F_MERGED) || include_unmerged)) continue;   /* mergeProcessed (:519-560) */
        if (dedupOut) continue;                                                      /* :575 */
        if (r1 && result1 == FP_PASS_FILTER && r2 && result2 == FP_PASS_FILTER) {
            /* :577-593: out1 / out2 */
        } else if (r1 && result1 == FP_PASS_FILTER) {                               /* :594-603 */
            if (unpairedLeft) {
                if (toUnpaired1) append_or(out, out_cap, &o, &or1, NULL);
                if (toFailed) append_or(out, out_cap, &o, &or2, FAILED_TYPES[result2]);
            } else if (toFailed) {
                append_or(out, out_cap, &o, &or1, "paired_read_is_failing");
                append_or(out, out_cap, &o, &or2, FAILED_TYPES[result2]);
            }
        } else if (r2 && result2 == FP_PASS_FILTER) {                               /* :604-619 */
            if (unpairedRight) {
                if (toUnpaired2) append_or(out, out_cap, &o, &or2, NULL);
                if (toFailed) append_or(out, out_cap, &o, &or1, FAILED_TYPES[result1]);
            } else if (unpairedLeft) {
                if (toUnpaired1) append_or(out, out_cap, &o, &or2, NULL);
                if (toFailed) append_or(out, out_cap, &o, &or1, FAILED_TYPES[result1]);
            } else if (toFailed) {
                append_or(out, out_cap, &o, &or1, FAILED_TYPES[result1]);
                append_or(out, out_cap, &o, &or2, "paired_read_is_failing");
            }
        }
    }
    return o;
}
