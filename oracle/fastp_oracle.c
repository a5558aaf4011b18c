/*
 * fastp_oracle.c -- CPU restatement ("port") of the reference's per-read hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may call this.  The product (libfastp_b200.so) never links or loads it.
 *
 * Plain scalar C, one function per reference function, each citing the reference file:line it
 * follows (OpenGene/fastp v1.3.6 under /root/reference).  Parity status: PINNED -- this port is
 * checked (tests/test_oracle_vs_reference.py, run where /root/reference exists) against the
 * reference's own objects compiled into oracle/_ref/libfastp_ref.so, against the reference's
 * unit-test vectors (tests/test_oracle_kat.py) and against golden fixtures generated from the
 * reference build (tests/golden/).
 *
 * Parity domain: bases in {A,C,G,T,N}, quals in [33,126] (SURVEY.md 8c).
 */
#include "fastp_oracle.h"
#include <stdlib.h>
#include <string.h>

typedef struct {
    uint8_t* seq;   /* points INTO the batch row, advanced by frontTrimmed (string::erase(0,front)) */
    uint8_t* qual;
    int len;
    int is_null;    /* trimAndCut returned NULL */
} oread;

static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* util.h:16-33 */
static inline uint8_t complement(uint8_t base) {
    switch (base) {
        case 'A': case 'a': return 'T';
        case 'T': case 't': return 'A';
        case 'C': case 'c': return 'G';
        case 'G': case 'g': return 'C';
        default: return 'N';
    }
}

/* Read::resize src/read.cpp:62-67 */
static inline void read_resize(oread* r, int len) {
    if (len > r->len || len < 0) return;
    r->len = len;
}

/* ------------------------------------------------------------------------------------------
 * Stats::statRead per-base part  src/stats.cpp:191-268 (+ :290 mReads++)
 * ------------------------------------------------------------------------------------------ */
static inline int base2val(uint8_t b) {  /* stats.cpp:293-318 */
    switch (b) { case 'A': return 0; case 'T': return 1; case 'C': return 2; case 'G': return 3; default: return -1; }
}

/* mOverRepSeq (stats.h:91) is a std::map<string, long>: its keys ordered by bytes, looked up in O(log K).  Restated as the candidates
 * of each side sorted by (bytes, index); a window is found by binary search, the lowest index among equal strings wins (the lists
 * are duplicate-free, as the map's keys are, so that tie never arises in practice). */
typedef struct { const char* s; int len, k; } ovr_key;
typedef struct { ovr_key* keys[2]; int K[2]; } ovr_index;

static int ovr_key_cmp(const void* a, const void* b) {
    const ovr_key *x = (const ovr_key*)a, *y = (const ovr_key*)b;
    const int c = strcmp(x->s, y->s);
    return c ? c : (x->k > y->k) - (x->k < y->k);
}

static int ovr_index_make(ovr_index* X, const fp_params* p, const fp_counter_layout* L) {
    memset(X, 0, sizeof(*X));
    if (!p->overrep_enabled) return 1;
    for (int side = 0; side < 2; side++) {
        const int K = L->n_overrep[side];
        const char* const* cands = side ? p->overrep_seqs2 : p->overrep_seqs1;
        if (K <= 0) continue;
        X->keys[side] = (ovr_key*)malloc((size_t)K * sizeof(ovr_key));
        if (!X->keys[side]) return 0;
        for (int k = 0; k < K; k++) { X->keys[side][k].s = cands[k]; X->keys[side][k].len = (int)strlen(cands[k]); X->keys[side][k].k = k; }
        qsort(X->keys[side], (size_t)K, sizeof(ovr_key), ovr_key_cmp);
        X->K[side] = K;
    }
    return 1;
}

static void ovr_index_free(ovr_index* X) { free(X->keys[0]); free(X->keys[1]); }

/* byte order of the window w[0, n) against key c (a shorter string that is a prefix of the other comes first) */
static int ovr_window_cmp(const uint8_t* w, int n, const ovr_key* c) {
    const int m = imin(n, c->len);
    const int r = memcmp(w, c->s, (size_t)m);
    return r ? r : (n > c->len) - (n < c->len);
}

/* mOverRepSeq.count(seq) > 0: index of the candidate equal to w[0, n), -1 if none */
static int ovr_find(const ovr_index* X, int side, const uint8_t* w, int n) {
    if (n < 0) return -1;                                              /* step 5 of seq_len < 2: outside the domain (fp_params) */
    int lo = 0, hi = X->K[side];                                       /* lower bound of w in (bytes, index) order */
    while (lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        if (ovr_window_cmp(w, n, &X->keys[side][mid]) > 0) lo = mid + 1; else hi = mid;
    }
    return lo < X->K[side] && ovr_window_cmp(w, n, &X->keys[side][lo]) == 0 ? X->keys[side][lo].k : -1;
}

static void stat_read(const fp_params* p, const ovr_index* X, int64_t* C, const fp_counter_layout* L, int s, const uint8_t* seq, const uint8_t* qual, int len) {
    C[fp_off_length_sum(L, s)] += len;                                  /* stats.cpp:194 */
    int kmer = 0;
    int needFullCompute = 1;
    for (int i = 0; i < len; i++) {
        uint8_t base = seq[i];
        uint8_t q = qual[i];
        int b = base & 0x07;                                            /* stats.cpp:208 */
        if (q < FP_QUAL_BINS) C[fp_off_qualhist(L, s, q)]++;            /* stats.cpp:213 */
        if (i < L->cycles) {
            if (q >= '?') {                                             /* stats.cpp:215-220 */
                C[fp_off_cycle(L, s, 0 * 8 + b, i)]++;
                C[fp_off_cycle(L, s, 1 * 8 + b, i)]++;
            } else if (q >= '5') {
                C[fp_off_cycle(L, s, 1 * 8 + b, i)]++;
            }
            C[fp_off_cycle(L, s, 2 * 8 + b, i)]++;                      /* stats.cpp:222 */
            C[fp_off_cycle(L, s, 3 * 8 + b, i)] += (int)q - 33;         /* stats.cpp:223 */
            C[fp_off_cycle(L, s, 32, i)]++;                             /* stats.cpp:225 */
            C[fp_off_cycle(L, s, 33, i)] += (int)q - 33;                /* stats.cpp:226 */
        }
        if (base == 'N') { needFullCompute = 1; continue; }             /* stats.cpp:228-231 */
        if (i < 4) continue;                                            /* stats.cpp:234-235 */
        if (!needFullCompute) {                                         /* stats.cpp:239-247 */
            int val = base2val(base);
            if (val < 0) { needFullCompute = 1; continue; }
            kmer = ((kmer << 2) & 0x3FC) | val;
            C[fp_off_kmer(L, s, kmer)]++;
        } else {                                                        /* stats.cpp:248-265 */
            int valid = 1;
            kmer = 0;
            for (int k = 0; k < 5; k++) {
                int val = base2val(seq[i - 4 + k]);
                if (val < 0) { valid = 0; break; }
                kmer = ((kmer << 2) & 0x3FC) | val;
            }
            if (!valid) { needFullCompute = 1; continue; }
            C[fp_off_kmer(L, s, kmer)]++;
            needFullCompute = 0;
        }
    }
    /* over-representation analysis for 1 of every `sampling` reads  stats.cpp:270-288 */
    if (p->overrep_enabled) {
        if (C[fp_off_reads(L, s)] % p->overrep_sampling == 0) {
            const int side = s >> 1;
            const int evalLen = L->overrep_len[side];
            const int steps[5] = {10, 20, 40, 100, imin(150, evalLen - 2)};
            for (int s5 = 0; s5 < 5; s5++) {
                const int step = steps[s5];
                for (int i = 0; i < len - step; i++) {
                    const int hit = ovr_find(X, side, seq + i, step);  /* mOverRepSeq.count(seq) > 0 */
                    if (hit >= 0) {
                        C[fp_off_overrep_count(L, s, hit)]++;
                        for (int q = i; q < step + i && q < evalLen; q++) C[fp_off_overrep_dist(L, s, hit, q)]++;
                        i += step;
                    }
                }
            }
        }
    }
    C[fp_off_reads(L, s)]++;                                            /* stats.cpp:290 */
}

/* ------------------------------------------------------------------------------------------
 * Filter::trimAndCut  src/filter.cpp:68-207.   Returns 0 = NULL, 1 = read kept (mutated in place).
 * ------------------------------------------------------------------------------------------ */
static int trim_and_cut(const fp_params* p, oread* r, int front, int tail, int* frontTrimmed) {
    *frontTrimmed = 0;
    int anycut = p->cut_front || p->cut_tail || p->cut_right;
    if (front == 0 && tail == 0 && !anycut) return 1;                   /* filter.cpp:71-72 */

    int rlen = r->len - front - tail;                                   /* filter.cpp:75 */
    if (rlen < 0) return 0;

    if (front == 0 && !anycut) {                                        /* filter.cpp:79-81 */
        read_resize(r, rlen);
        return 1;
    } else if (!anycut) {                                               /* filter.cpp:82-89 */
        /* string::erase(0,front) then resize(rlen) */
        r->seq += front; r->qual += front; r->len = rlen;
        *frontTrimmed = front;
        return 1;
    }

    int l = r->len;
    const signed char* qualstr = (const signed char*)r->qual;
    const uint8_t* seq = r->seq;

    if (p->cut_front) {                                                 /* filter.cpp:97-127 */
        int w = p->cut_front_window;
        int s = front;
        if (l - front - tail - w <= 0) return 0;
        int totalQual = 0;
        for (int i = 0; i < w - 1; i++) totalQual += qualstr[s + i];
        for (s = front; s + w < l - tail; s++) {
            totalQual += qualstr[s + w - 1];
            if (s > front) totalQual -= qualstr[s - 1];
            if (totalQual >= w * (33 + p->cut_front_quality)) break;
        }
        if (s > 0) s = s + w - 1;
        while (s < l && seq[s] == 'N') s++;
        front = s;
        rlen = l - front - tail;
    }

    if (p->cut_right) {                                                 /* filter.cpp:130-163 */
        int w = p->cut_right_window;
        int s = front;
        if (l - front - tail - w <= 0) return 0;
        int totalQual = 0;
        for (int i = 0; i < w - 1; i++) totalQual += qualstr[s + i];
        int foundLowQualWindow = 0;
        for (s = front; s + w < l - tail; s++) {
            totalQual += qualstr[s + w - 1];
            if (s > front) totalQual -= qualstr[s - 1];
            if (totalQual < w * (33 + p->cut_right_quality)) { foundLowQualWindow = 1; break; }
        }
        if (foundLowQualWindow) {
            while (s < l - 1 && qualstr[s] >= 33 + p->cut_right_quality) s++;
            rlen = s - front;
        }
    }

    if (!p->cut_right && p->cut_tail) {                                 /* filter.cpp:166-194 */
        int w = p->cut_tail_window;
        if (l - front - tail - w <= 0) return 0;
        int totalQual = 0;
        int t = l - tail - 1;
        for (int i = 0; i < w - 1; i++) totalQual += qualstr[t - i];
        for (t = l - tail - 1; t - w >= front; t--) {
            totalQual += qualstr[t - w + 1];
            if (t < l - tail - 1) totalQual -= qualstr[t + 1];
            if (totalQual >= w * (33 + p->cut_tail_quality)) break;
        }
        if (t < l - 1) t = t - w + 1;
        while (t >= 0 && seq[t] == 'N') t--;
        rlen = t - front + 1;
    }

    if (rlen <= 0 || front >= l - 1) return 0;                          /* filter.cpp:196-197 */

    r->seq += front; r->qual += front; r->len = rlen;                   /* filter.cpp:199-202 */
    *frontTrimmed = front;
    return 1;
}

/* ------------------------------------------------------------------------------------------
 * PolyX::trimPolyG  src/polyx.cpp:16-42
 * ------------------------------------------------------------------------------------------ */
static int trim_polyg(oread* r, int compareReq) {
    const int allowOneMismatchForEach = 8;
    const int maxMismatch = 5;
    const uint8_t* data = r->seq;
    int rlen = r->len;
    int mismatch = 0;
    int i = 0;
    int firstGPos = rlen - 1;
    for (i = 0; i < rlen; i++) {
        if (data[rlen - i - 1] != 'G') mismatch++;
        else firstGPos = rlen - i - 1;
        int allowedMismatch = (i + 1) / allowOneMismatchForEach;
        if (mismatch > maxMismatch || (mismatch > allowedMismatch && i >= compareReq - 1)) break;
    }
    if (i >= compareReq) {
        int before = r->len;
        read_resize(r, firstGPos);
        return r->len != before;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * PolyX::trimPolyX  src/polyx.cpp:49-116.  Returns 1 if addPolyXTrimmed was called.
 * data[-1] (read when the scan consumed the whole read, polyx.cpp:107) is the byte before the
 * std::string buffer in the reference -- never a base letter; modelled as "does not match".
 * ------------------------------------------------------------------------------------------ */
static int trim_polyx(oread* r, int compareReq, int* polyOut, int* lenOut) {
    const int allowOneMismatchForEach = 8;
    const int maxMismatch = 5;
    const uint8_t* data = r->seq;
    int rlen = r->len;
    int atcgNumbers[4] = {0, 0, 0, 0};
    int pos = 0;
    for (pos = 0; pos < rlen; pos++) {
        uint8_t c = data[rlen - pos - 1];
        switch (c) {                                                    /* POLYX_BASE_IDX polyx.cpp:59-69 */
            case 'A': atcgNumbers[0]++; break;
            case 'T': atcgNumbers[1]++; break;
            case 'C': atcgNumbers[2]++; break;
            case 'G': atcgNumbers[3]++; break;
            case 'N': atcgNumbers[0]++; atcgNumbers[1]++; atcgNumbers[2]++; atcgNumbers[3]++; break;
            default: break;
        }
        int cmp = pos + 1;
        int allowedMismatch = imin(maxMismatch, cmp / allowOneMismatchForEach);
        int needToBreak = 1;
        for (int b = 0; b < 4; b++)
            if (cmp - atcgNumbers[b] <= allowedMismatch) needToBreak = 0;
        if (needToBreak && (pos >= allowOneMismatchForEach || pos + 1 >= compareReq - 1)) break;
    }
    if (pos + 1 >= compareReq) {                                        /* polyx.cpp:96-115 */
        int poly = 0;
        int maxCount = -1;
        for (int b = 0; b < 4; b++)
            if (atcgNumbers[b] > maxCount) { maxCount = atcgNumbers[b]; poly = b; }
        static const uint8_t ATCG[4] = {'A', 'T', 'C', 'G'};            /* common.h:25 */
        uint8_t polyBase = ATCG[poly];
        for (;;) {                                                      /* polyx.cpp:107-108 */
            int idx = rlen - pos - 1;
            uint8_t c = (idx < 0 || idx >= rlen) ? 0 : data[idx];       /* data[-1] / data[rlen]=='\0' */
            if (c != polyBase && pos >= 0) pos--; else break;
        }
        read_resize(r, rlen - pos - 1);
        *polyOut = poly;
        *lenOut = pos + 1;
        return 1;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * fastp_simd scalar restatements  src/simd.cpp:281-324
 * ------------------------------------------------------------------------------------------ */
static void reverse_complement(const uint8_t* src, uint8_t* dst, int len) {   /* simd.cpp:297-310 */
    for (int i = 0; i < len; i++) dst[len - 1 - i] = complement(src[i]);
}
static int count_mismatches(const uint8_t* a, const uint8_t* b, int len) {    /* simd.cpp:320-324 */
    int d = 0;
    for (int i = 0; i < len; i++) if (a[i] != b[i]) d++;
    return d;
}

/* ------------------------------------------------------------------------------------------
 * OverlapAnalysis::analyze  src/overlapanalysis.cpp:17-146 (allowGap=false passes only)
 * ------------------------------------------------------------------------------------------ */
static int diff_with_one_insertion(const uint8_t* insData, const uint8_t* normalData, int cmplen, int diffLimit);

static fp_ov_result analyze(const oread* r1, const oread* r2, int diffLimit, int overlapRequire, double diffPercentLimit, int allowGap) {
    uint8_t rcr2[FP_MAX_STRIDE + 8];
    int len2 = r2->len;
    reverse_complement(r2->seq, rcr2, len2);
    int len1 = r1->len;
    const uint8_t* str1 = r1->seq;
    const uint8_t* str2 = rcr2;
    const int complete_compare_require = 50;
    int overlap_len = 0, offset = 0, diff = 0;
    fp_ov_result ov;
    memset(&ov, 0, sizeof(ov));

    /* forward: overlapanalysis.cpp:48-65 */
    while (offset < len1 - overlapRequire) {
        overlap_len = imin(len1 - offset, len2);
        int overlapDiffLimit = imin(diffLimit, (int)(overlap_len * diffPercentLimit));
        int protectedPrefix = imin(overlap_len, complete_compare_require);       /* :34-44 */
        diff = count_mismatches(str1 + offset, str2, protectedPrefix);
        if (diff <= overlapDiffLimit) {
            if (overlap_len > complete_compare_require) diff = count_mismatches(str1 + offset, str2, overlap_len);
            ov.overlapped = 1; ov.offset = (int16_t)offset; ov.overlap_len = (int16_t)overlap_len; ov.diff = (int16_t)diff; ov.has_gap = 0;
            return ov;
        }
        offset += 1;
    }
    /* reverse: overlapanalysis.cpp:73-89 */
    offset = 0;
    while (offset > -(len2 - overlapRequire)) {
        overlap_len = imin(len1, len2 - abs(offset));
        int overlapDiffLimit = imin(diffLimit, (int)(overlap_len * diffPercentLimit));
        int protectedPrefix = imin(overlap_len, complete_compare_require);
        diff = count_mismatches(str1, str2 + (-offset), protectedPrefix);
        if (diff <= overlapDiffLimit) {
            if (overlap_len > complete_compare_require) diff = count_mismatches(str1, str2 + (-offset), overlap_len);
            ov.overlapped = 1; ov.offset = (int16_t)offset; ov.overlap_len = (int16_t)overlap_len; ov.diff = (int16_t)diff; ov.has_gap = 0;
            return ov;
        }
        offset -= 1;
    }
    if (allowGap) {
        /* forward with one gap: overlapanalysis.cpp:91-114 */
        offset = 0;
        while (offset < len1 - overlapRequire) {
            overlap_len = imin(len1 - offset, len2);
            int overlapDiffLimit = imin(diffLimit, (int)(overlap_len * diffPercentLimit));
            int d = diff_with_one_insertion(str1 + offset, str2, overlap_len - 1, overlapDiffLimit);
            if (d < 0 || d > overlapDiffLimit) d = diff_with_one_insertion(str2, str1 + offset, overlap_len - 1, overlapDiffLimit);
            if (d <= overlapDiffLimit && d >= 0) {
                ov.overlapped = 1; ov.offset = (int16_t)offset; ov.overlap_len = (int16_t)overlap_len; ov.diff = (int16_t)d; ov.has_gap = 1;
                return ov;
            }
            offset += 1;
        }
        /* reverse with one gap: overlapanalysis.cpp:116-138 */
        offset = 0;
        while (offset > -(len2 - overlapRequire)) {
            overlap_len = imin(len1, len2 - abs(offset));
            int overlapDiffLimit = imin(diffLimit, (int)(overlap_len * diffPercentLimit));
            int d = diff_with_one_insertion(str1, str2 - offset, overlap_len - 1, overlapDiffLimit);
            if (d < 0 || d > overlapDiffLimit) d = diff_with_one_insertion(str2 - offset, str1, overlap_len - 1, overlapDiffLimit);
            if (d <= overlapDiffLimit && d >= 0) {
                ov.overlapped = 1; ov.offset = (int16_t)offset; ov.overlap_len = (int16_t)overlap_len; ov.diff = (int16_t)d; ov.has_gap = 1;
                return ov;
            }
            offset -= 1;
        }
    }
    return ov;                                                          /* :141-145 all zero */
}

/* ------------------------------------------------------------------------------------------
 * BaseCorrector::correctByOverlapAnalysis  src/basecorrector.cpp:21-83
 * ------------------------------------------------------------------------------------------ */
static int correct_by_overlap(oread* r1, oread* r2, int64_t* FR, fp_ov_result ov, int* r1c, int* r2c) {
    *r1c = *r2c = 0;
    if (ov.diff == 0 || !ov.overlapped) return 0;                       /* :23-24 */
    int ol = ov.overlap_len;
    int start1 = imax(0, ov.offset);
    int start2 = r2->len - imax(0, -ov.offset) - 1;
    uint8_t* seq1 = r1->seq; uint8_t* seq2 = r2->seq;
    uint8_t* qual1 = r1->qual; uint8_t* qual2 = r2->qual;
    const signed char GOOD_QUAL = 33 + 30, BAD_QUAL = 33 + 14;          /* num2qual(30), num2qual(14) */
    int corrected = 0;
    for (int i = 0; i < ol; i++) {
        int p1 = start1 + i;
        int p2 = start2 - i;
        if (seq1[p1] != complement(seq2[p2])) {
            if ((signed char)qual1[p1] >= GOOD_QUAL && (signed char)qual2[p2] <= BAD_QUAL) {
                seq2[p2] = complement(seq1[p1]);                        /* :44-45 */
                qual2[p2] = qual1[p1];
                corrected++; *r2c = 1;
                /* :49 addCorrection(seq2[p2], complement(seq1[p1])) reads the ALREADY OVERWRITTEN seq2[p2]
                   (c_str alias) => from == to: only the diagonal is ever incremented (SURVEY App. A.6) */
                FR[FP_FR_CORRECTION + (seq2[p2] & 7) * 8 + (complement(seq1[p1]) & 7)]++;
            } else if ((signed char)qual2[p2] >= GOOD_QUAL && (signed char)qual1[p1] <= BAD_QUAL) {
                seq1[p1] = complement(seq2[p2]);                        /* :53-54 */
                qual1[p1] = qual2[p2];
                corrected++; *r1c = 1;
                FR[FP_FR_CORRECTION + (seq1[p1] & 7) * 8 + (complement(seq2[p2]) & 7)]++;
            }
        }
    }
    if (corrected > 0) FR[FP_FR_CORRECTED_READS] += (*r1c && *r2c) ? 2 : 1;   /* :75-80 */
    return corrected;
}

/* ------------------------------------------------------------------------------------------
 * Matcher::matchWithOneInsertion  src/matcher.cpp:10-54 (literal restatement; arrays zero-filled
 * where the reference leaves VLAs uninitialised -- those elements are never read, see matcher.cpp:46-47)
 * ------------------------------------------------------------------------------------------ */
static int match_with_one_insertion(const uint8_t* insData, const uint8_t* normalData, int cmplen, int diffLimit) {
    int accL[FP_MAX_STRIDE + 8];
    int accR[FP_MAX_STRIDE + 8];
    if (cmplen <= 0) return 0;
    memset(accL, 0, sizeof(int) * cmplen);
    memset(accR, 0, sizeof(int) * cmplen);
    accL[0] = insData[0] == normalData[0] ? 0 : 1;
    accR[cmplen - 1] = insData[cmplen] == normalData[cmplen - 1] ? 0 : 1;
    for (int i = 1; i < cmplen; i++) {
        if (insData[i] != normalData[i]) accL[i] = accL[i - 1] + 1;
        else accL[i] = accL[i - 1];
        if (accL[i] + accR[cmplen - 1] > diffLimit) break;
    }
    for (int i = cmplen - 2; i >= 0; i--) {
        if (insData[i + 1] != normalData[i]) accR[i] = accR[i + 1] + 1;
        else accR[i] = accR[i + 1];
        if (accR[i] + accL[0] > diffLimit) {
            for (int q = 0; q < i; q++) accR[q] = diffLimit + 1;
            break;
        }
    }
    for (int i = 1; i < cmplen; i++) {
        if (accL[i - 1] + accR[cmplen - 1] > diffLimit) return 0;
        int diff = accL[i - 1] + accR[i];
        if (diff <= diffLimit) return 1;
    }
    return 0;
}

/* Matcher::diffWithOneInsertion  src/matcher.cpp:56-100 (literal restatement, arrays zero-filled) */
static int diff_with_one_insertion(const uint8_t* insData, const uint8_t* normalData, int cmplen, int diffLimit) {
    int accL[FP_MAX_STRIDE + 8];
    int accR[FP_MAX_STRIDE + 8];
    if (cmplen <= 0) return 100000000;
    memset(accL, 0, sizeof(int) * cmplen);
    memset(accR, 0, sizeof(int) * cmplen);
    accL[0] = insData[0] == normalData[0] ? 0 : 1;
    accR[cmplen - 1] = insData[cmplen] == normalData[cmplen - 1] ? 0 : 1;
    for (int i = 1; i < cmplen; i++) {
        if (insData[i] != normalData[i]) accL[i] = accL[i - 1] + 1;
        else accL[i] = accL[i - 1];
        if (accL[i] + accR[cmplen - 1] > diffLimit) break;
    }
    for (int i = cmplen - 2; i >= 0; i--) {
        if (insData[i + 1] != normalData[i]) accR[i] = accR[i + 1] + 1;
        else accR[i] = accR[i + 1];
        if (accR[i] + accL[0] > diffLimit) {
            for (int q = 0; q < i; q++) accR[q] = diffLimit + 1;
            break;
        }
    }
    int minDiff = 100000000;
    for (int i = 1; i < cmplen; i++) {
        if (accL[i - 1] + accR[cmplen - 1] > diffLimit) return -1;
        int diff = accL[i - 1] + accR[i];
        if (diff <= minDiff) minDiff = diff;
    }
    return minDiff;
}

/* ------------------------------------------------------------------------------------------
 * AdapterTrimmer::trimBySequence  src/adaptertrimmer.cpp:64-157
 * Returns 1 if trimmed. *posOut = hit position, *basesOut = adapter bases counted by
 * FilterResult::addAdapterTrimmed(adapter,isR2) (filterresult.cpp:124-128: empty adapter adds nothing).
 * ------------------------------------------------------------------------------------------ */
static int trim_by_sequence(oread* r, int64_t* FR, const char* adapterseq, int matchReq, int* posOut, int* basesOut) {
    const int allowOneMismatchForEach = 8;
    int rlen = r->len;
    int alen = (int)strlen(adapterseq);
    const uint8_t* adata = (const uint8_t*)adapterseq;
    const uint8_t* rdata = r->seq;
    if (alen < matchReq) return 0;                                      /* :73-74 */
    int pos = 0, found = 0, start = 0;
    if (alen >= 16) start = -4; else if (alen >= 12) start = -3; else if (alen >= 8) start = -2;
    for (pos = start; pos < rlen - matchReq; pos++) {                   /* :87-100 */
        int cmplen = imin(rlen - pos, alen);
        int allowedMismatch = cmplen / allowOneMismatchForEach;
        int startOffset = imax(0, -pos);
        int mismatch = count_mismatches(adata + startOffset, rdata + startOffset + pos, cmplen - startOffset);
        if (mismatch <= allowedMismatch) { found = 1; break; }
    }
    if (!found) {                                                       /* :105-118 insertion */
        for (pos = 0; pos < rlen - matchReq - 1; pos++) {
            int cmplen = imin(rlen - pos - 1, alen);
            int allowedMismatch = cmplen / allowOneMismatchForEach - 1;
            /* rdata is NOT advanced by pos (adaptertrimmer.cpp:110) */
            if (match_with_one_insertion(rdata, adata, cmplen, allowedMismatch)) { found = 1; break; }
        }
    }
    if (!found) {                                                       /* :122-135 deletion */
        for (pos = 0; pos < rlen - matchReq; pos++) {
            int cmplen = imin(rlen - pos, alen - 1);
            int allowedMismatch = cmplen / allowOneMismatchForEach - 1;
            if (match_with_one_insertion(adata, rdata, cmplen, allowedMismatch)) { found = 1; break; }
        }
    }
    if (found) {                                                        /* :137-154 */
        int abases;
        if (pos < 0) {
            abases = alen + pos;                                        /* adapterseq.substr(0, alen+pos) */
            r->len = 0;
        } else {
            abases = rlen - pos;                                        /* mSeq->substr(pos, rlen-pos) */
            read_resize(r, pos);
        }
        if (abases > 0) FR[FP_FR_ADAPTER_BASES] += abases;              /* filterresult.cpp:124-127 */
        *posOut = pos; *basesOut += imax(abases, 0);
        return 1;
    }
    return 0;
}

/* AdapterTrimmer::trimByMultiSequences  src/adaptertrimmer.cpp:48-62 */
static int trim_by_multi(const fp_params* p, oread* r, int64_t* FR, int* posOut, int* basesOut) {
    int matchReq = 4;
    if (p->n_fasta_adapters > 16) matchReq = 5;
    if (p->n_fasta_adapters > 256) matchReq = 6;
    int trimmed = 0;
    for (int i = 0; i < p->n_fasta_adapters; i++)
        trimmed |= trim_by_sequence(r, FR, p->fasta_adapters[i], matchReq, posOut, basesOut);
    return trimmed;
}

/* ------------------------------------------------------------------------------------------
 * Filter::passFilter  src/filter.cpp:15-57 (+ countQualityMetrics simd.cpp:281-295,
 * passLowComplexityFilter filter.cpp:59-66, countAdjacentDiffs simd.cpp:312-318)
 * ------------------------------------------------------------------------------------------ */
static int pass_filter(const fp_params* p, const oread* r) {
    if (r->is_null || r->len == 0) return FP_FAIL_LENGTH;
    int rlen = r->len;
    int lowQualNum = 0, nBaseNum = 0, totalQual = 0;
    if (p->qual_filter_enabled || p->length_filter_enabled) {
        for (int i = 0; i < rlen; i++) {
            uint8_t q = r->qual[i];
            totalQual += q - 33;
            if (q < (uint8_t)p->qualified_qual) lowQualNum++;
            if (r->seq[i] == 'N') nBaseNum++;
        }
    }
    if (p->qual_filter_enabled) {
        if (lowQualNum > (p->unqualified_percent_limit * rlen / 100.0)) return FP_FAIL_QUALITY;
        else if (p->avg_qual_req > 0 && (totalQual / rlen) < p->avg_qual_req) return FP_FAIL_QUALITY;
        else if (nBaseNum > p->n_base_limit) return FP_FAIL_N_BASE;
    }
    if (p->length_filter_enabled) {
        if (rlen < p->length_required) return FP_FAIL_LENGTH;
        if (p->length_limit > 0 && rlen > p->length_limit) return FP_FAIL_TOO_LONG;
    }
    if (p->complexity_filter_enabled) {
        if (rlen <= 1) return FP_FAIL_COMPLEXITY;
        int diff = 0;
        for (int i = 0; i < rlen - 1; i++) if (r->seq[i] != r->seq[i + 1]) diff++;
        if (!((double)diff / (double)(rlen - 1) >= p->complexity_threshold)) return FP_FAIL_COMPLEXITY;
    }
    return FP_PASS_FILTER;
}

static void fill_result(fp_read_result* o, const oread* r, const uint8_t* row, int verdict, int pair_verdict,
                        int flags, int apos, int abases, int polyBase, int polyLen) {
    memset(o, 0, sizeof(*o));
    if (r->is_null) { o->front = 0; o->len = 0; flags |= FP_F_DROPPED; }
    else { o->front = (uint16_t)(r->seq - row); o->len = (uint16_t)r->len; }
    o->verdict = (uint8_t)verdict;
    o->pair_verdict = (uint8_t)pair_verdict;
    o->flags = (uint8_t)flags;
    o->adapter_pos = (int16_t)apos;
    o->adapter_len = (uint16_t)abases;
    o->polyx_base = (uint8_t)polyBase;
    o->polyx_len = (uint16_t)polyLen;
}

/* ------------------------------------------------------------------------------------------
 * SingleEndProcessor::processSingleEnd loop body  src/seprocessor.cpp:204-296
 * ------------------------------------------------------------------------------------------ */
static void process_se_one(const fp_params* p, const ovr_index* X, const fp_counter_layout* L, int64_t* C,
                           uint8_t* seq, uint8_t* qual, int len, int dedupOut, fp_read_result* out) {
    int64_t* FR = C + L->off_filter;
    stat_read(p, X, C, L, FP_STATS_PRE1, seq, qual, len);                     /* :211 */
    oread r = {seq, qual, len, 0};
    int frontTrimmed = 0, flags = dedupOut ? FP_F_DUPLICATE : 0, apos = 0, abases = 0, polyBase = 255, polyLen = 0;
    if (!trim_and_cut(p, &r, p->trim_front1, p->trim_tail1, &frontTrimmed)) r.is_null = 1;   /* :235 */
    if (!r.is_null && p->polyg_enabled)                                 /* :237-240 */
        if (trim_polyg(&r, p->polyg_min_len)) flags |= FP_F_POLYG_TRIMMED;
    int isAdapterDimer = 0;
    if (!r.is_null && p->adapter_enabled) {                             /* :243-260 */
        int trimmed = 0;
        if (p->has_seq_r1) trimmed = trim_by_sequence(&r, FR, p->adapter_seq_r1, 4, &apos, &abases);
        if (p->n_fasta_adapters > 0) trimmed |= trim_by_multi(p, &r, FR, &apos, &abases);
        if (trimmed) { FR[FP_FR_ADAPTER_READS] += 1; flags |= FP_F_ADAPTER_TRIMMED; }
        if (trimmed && r.len <= p->dimer_max_len) isAdapterDimer = 1;
    }
    if (!r.is_null && p->polyx_enabled) {                               /* :263-266 */
        if (trim_polyx(&r, p->polyx_min_len, &polyBase, &polyLen)) {
            FR[FP_FR_POLYX_READS + polyBase] += 1;                      /* filterresult.cpp:186-189 */
            FR[FP_FR_POLYX_BASES + polyBase] += polyLen;
            flags |= FP_F_POLYX_TRIMMED;
        }
    }
    if (!r.is_null) {                                                   /* :268-271 */
        if (p->max_len1 > 0 && p->max_len1 < r.len) read_resize(&r, p->max_len1);
    }
    int result = pass_filter(p, &r);                                    /* :273 */
    if (isAdapterDimer) { result = FP_FAIL_ADAPTER_DIMER; flags |= FP_F_ADAPTER_DIMER; }   /* :275-276 */
    FR[FP_FR_READSTATS + result] += 1;                                  /* :278 */
    if (!dedupOut && !r.is_null && result == FP_PASS_FILTER)            /* :280-286 */
        stat_read(p, X, C, L, FP_STATS_POST1, r.seq, r.qual, r.len);
    fill_result(out, &r, seq, result, result, flags, apos, abases, polyBase, polyLen);
}

/* ------------------------------------------------------------------------------------------
 * PairEndProcessor::processPairEnd loop body  src/peprocessor.cpp:383-643 (incl. merging mode :519-560 and dedupOut :397-401;
 * no overlapped_out / index filter / UMI) + statInsertSize :710-723
 * ------------------------------------------------------------------------------------------ */
static void process_pe_one(const fp_params* p, const ovr_index* X, const fp_counter_layout* L, int64_t* C,
                           uint8_t* seq1, uint8_t* qual1, int len1, uint8_t* seq2, uint8_t* qual2, int len2, int dedupOut,
                           fp_read_result* out1, fp_read_result* out2, fp_ov_result* ovOut) {
    int64_t* FR = C + L->off_filter;
    int64_t* ISZ = C + L->off_isize;
    stat_read(p, X, C, L, FP_STATS_PRE1, seq1, qual1, len1);                  /* :393-394 */
    stat_read(p, X, C, L, FP_STATS_PRE2, seq2, qual2, len2);
    oread r1 = {seq1, qual1, len1, 0}, r2 = {seq2, qual2, len2, 0};
    int ft1 = 0, ft2 = 0;
    int flags1 = dedupOut ? FP_F_DUPLICATE : 0, flags2 = flags1, apos1 = 0, apos2 = 0, ab1 = 0, ab2 = 0, pb1 = 255, pb2 = 255, pl1 = 0, pl2 = 0;
    if (!trim_and_cut(p, &r1, p->trim_front1, p->trim_tail1, &ft1)) r1.is_null = 1;   /* :425-426 */
    if (!trim_and_cut(p, &r2, p->trim_front2, p->trim_tail2, &ft2)) r2.is_null = 1;
    int both = !r1.is_null && !r2.is_null;
    if (both && p->polyg_enabled) {                                     /* :428-431 */
        if (trim_polyg(&r1, p->polyg_min_len)) flags1 |= FP_F_POLYG_TRIMMED;
        if (trim_polyg(&r2, p->polyg_min_len)) flags2 |= FP_F_POLYG_TRIMMED;
    }
    int isizeEvaluated = 0, isAdapterDimer = 0;
    fp_ov_result ov; memset(&ov, 0, sizeof(ov));
    int ovComputed = 0;
    if (both && (p->adapter_enabled || p->correction_enabled || p->thread0_semantics)) {   /* :438-441 */
        ov = analyze(&r1, &r2, p->overlap_diff_limit, p->overlap_require, p->overlap_diff_percent_limit / 100.0, 0);
        ovComputed = 1;
    }
    if (both && (p->adapter_enabled || p->correction_enabled)) {        /* :443 */
        /* :445-447 gap-aware adapter trimming computes a separate overlap */
        fp_ov_result ovForAdapter = p->allow_gap_overlap_trimming
            ? analyze(&r1, &r2, p->overlap_diff_limit, p->overlap_require, p->overlap_diff_percent_limit / 100.0, 1) : ov;
        if (p->thread0_semantics) {                                     /* :449-452 statInsertSize */
            int isize = p->insert_size_max;
            if (ov.overlapped) {
                if (ov.offset > 0) isize = r1.len + r2.len - ov.overlap_len + ft1 + ft2;
                else isize = ov.overlap_len + ft1 + ft2;
            }
            if (isize > p->insert_size_max) isize = p->insert_size_max;
            ISZ[isize]++;
            isizeEvaluated = 1;
        }
        if (p->correction_enabled && !ovForAdapter.has_gap) {             /* :453-456 */
            int c1, c2;
            correct_by_overlap(&r1, &r2, FR, ovForAdapter, &c1, &c2);
            if (c1) flags1 |= FP_F_CORRECTED;
            if (c2) flags2 |= FP_F_CORRECTED;
        }
        if (p->adapter_enabled) {                                       /* :457-485 */
            int trimmed = 0;
            /* AdapterTrimmer::trimByOverlapAnalysis adaptertrimmer.cpp:17-46 */
            if (ovForAdapter.overlapped && ovForAdapter.offset < 0) {
                int ol = ovForAdapter.overlap_len;
                int nl1 = imin(r1.len, ol + ft2);
                int nl2 = imin(r2.len, ol + ft1);
                int a1 = r1.len - nl1, a2 = r2.len - nl2;
                read_resize(&r1, nl1);
                read_resize(&r2, nl2);
                FR[FP_FR_ADAPTER_BASES] += a1 + a2;                     /* filterresult.cpp:153-155 */
                ab1 += a1; ab2 += a2;
                trimmed = 1;
            }
            int trimmed1 = trimmed, trimmed2 = trimmed;
            if (!trimmed) {                                             /* :461-466 */
                if (p->has_seq_r1) trimmed1 = trim_by_sequence(&r1, FR, p->adapter_seq_r1, 4, &apos1, &ab1);
                if (p->has_seq_r2) trimmed2 = trim_by_sequence(&r2, FR, p->adapter_seq_r2, 4, &apos2, &ab2);
            }
            if (p->n_fasta_adapters > 0) {                              /* :467-470 */
                trimmed1 |= trim_by_multi(p, &r1, FR, &apos1, &ab1);
                trimmed2 |= trim_by_multi(p, &r2, FR, &apos2, &ab2);
            }
            if (trimmed1) { FR[FP_FR_ADAPTER_READS] += 1; flags1 |= FP_F_ADAPTER_TRIMMED; }   /* :472-475 */
            if (trimmed2) { FR[FP_FR_ADAPTER_READS] += 1; flags2 |= FP_F_ADAPTER_TRIMMED; }
            if ((trimmed1 || trimmed2) && r1.len <= p->dimer_max_len && r2.len <= p->dimer_max_len)   /* :480-484 */
                isAdapterDimer = 1;
        }
    }
    if (p->thread0_semantics && !isizeEvaluated && both) {              /* :497-504 */
        if (!ovComputed) {
            ov = analyze(&r1, &r2, p->overlap_diff_limit, p->overlap_require, p->overlap_diff_percent_limit / 100.0, 0);
            ovComputed = 1;
        }
        int isize = p->insert_size_max;
        if (ov.overlapped) {
            if (ov.offset > 0) isize = r1.len + r2.len - ov.overlap_len + ft1 + ft2;
            else isize = ov.overlap_len + ft1 + ft2;
        }
        if (isize > p->insert_size_max) isize = p->insert_size_max;
        ISZ[isize]++;
        isizeEvaluated = 1;
    }
    if (both && p->polyx_enabled) {                                     /* :506-509 */
        if (trim_polyx(&r1, p->polyx_min_len, &pb1, &pl1)) {
            FR[FP_FR_POLYX_READS + pb1] += 1; FR[FP_FR_POLYX_BASES + pb1] += pl1; flags1 |= FP_F_POLYX_TRIMMED;
        }
        if (trim_polyx(&r2, p->polyx_min_len, &pb2, &pl2)) {
            FR[FP_FR_POLYX_READS + pb2] += 1; FR[FP_FR_POLYX_BASES + pb2] += pl2; flags2 |= FP_F_POLYX_TRIMMED;
        }
    }
    if (both) {                                                         /* :511-516 */
        if (p->max_len1 > 0 && p->max_len1 < r1.len) read_resize(&r1, p->max_len1);
        if (p->max_len2 > 0 && p->max_len2 < r2.len) read_resize(&r2, p->max_len2);
    }
    int result1, result2, pv;
    int mergeProcessed = 0;
    if (p->merge_enabled && both) {                                     /* :519-560 merging mode */
        /* :523 the overlap is always computed again on the trimmed reads */
        ov = analyze(&r1, &r2, p->overlap_diff_limit, p->overlap_require, p->overlap_diff_percent_limit / 100.0, 0);
        ovComputed = 1;
        if (ov.overlapped) {
            /* OverlapAnalysis::merge overlapanalysis.cpp:148-179: r1[0,len1) + reverseComplement(r2)[ol, ol+len2) */
            const int ol = ov.overlap_len;
            const int mlen1 = ol + imax(0, ov.offset);
            const int mlen2 = ov.offset > 0 ? r2.len - ol : 0;
            uint8_t mseq[2 * FP_MAX_STRIDE], mqual[2 * FP_MAX_STRIDE];
            memcpy(mseq, r1.seq, (size_t)mlen1); memcpy(mqual, r1.qual, (size_t)mlen1);
            for (int k = 0; k < mlen2; k++) {                           /* rr2[ol + k] = complement(r2[len2 - 1 - ol - k]), quality reversed */
                mseq[mlen1 + k] = complement(r2.seq[r2.len - 1 - ol - k]);
                mqual[mlen1 + k] = r2.qual[r2.len - 1 - ol - k];
            }
            oread m = {mseq, mqual, mlen1 + mlen2, 0};
            const int result = pass_filter(p, &m);                      /* :526 */
            FR[FP_FR_READSTATS + result] += 2;                          /* :527 */
            if (result == FP_PASS_FILTER) {                             /* :528-534: dedupOut is not consulted for a merged read */
                stat_read(p, X, C, L, FP_STATS_POST1, mseq, mqual, m.len);
                FR[FP_FR_MERGED_PAIRS] += 1;                            /* mergedCount -> addMergedPairs :694 */
            }
            result1 = result2 = pv = result;
            flags1 |= FP_F_MERGED; flags2 |= FP_F_MERGED;
            mergeProcessed = 1;
        } else if (p->merge_include_unmerged) {                         /* :537-560 */
            result1 = pass_filter(p, &r1);
            result2 = pass_filter(p, &r2);
            if (isAdapterDimer) {
                result1 = result2 = FP_FAIL_ADAPTER_DIMER;
                flags1 |= FP_F_ADAPTER_DIMER; flags2 |= FP_F_ADAPTER_DIMER;
            }
            FR[FP_FR_READSTATS + result1] += 1;
            if (result1 == FP_PASS_FILTER && !dedupOut) stat_read(p, X, C, L, FP_STATS_POST1, r1.seq, r1.qual, r1.len);   /* :547 */
            FR[FP_FR_READSTATS + result2] += 1;
            if (result2 == FP_PASS_FILTER && !dedupOut) stat_read(p, X, C, L, FP_STATS_POST1, r2.seq, r2.qual, r2.len);   /* :553; read 2 into read 1's Stats: :555 */
            pv = imax(result1, result2);
            mergeProcessed = 1;
        }
    }
    if (!mergeProcessed) {
        result1 = pass_filter(p, &r1);                                  /* :565-566 */
        result2 = pass_filter(p, &r2);
        if (isAdapterDimer) {                                           /* :568-571 */
            result1 = result2 = FP_FAIL_ADAPTER_DIMER;
            flags1 |= FP_F_ADAPTER_DIMER; flags2 |= FP_F_ADAPTER_DIMER;
        }
        pv = imax(result1, result2);
        FR[FP_FR_READSTATS + pv] += 2;                                  /* :573 */
        if (!dedupOut && !p->merge_enabled && !r1.is_null && result1 == FP_PASS_FILTER && !r2.is_null && result2 == FP_PASS_FILTER) {   /* :575-591 */
            stat_read(p, X, C, L, FP_STATS_POST1, r1.seq, r1.qual, r1.len);
            stat_read(p, X, C, L, FP_STATS_POST2, r2.seq, r2.qual, r2.len);
        }
    }
    fill_result(out1, &r1, seq1, result1, pv, flags1, apos1, ab1, pb1, pl1);
    fill_result(out2, &r2, seq2, result2, pv, flags2, apos2, ab2, pb2, pl2);
    if (ovOut) *ovOut = ov;
    (void)ovComputed;
}

int fp_oracle_process_dedup(const fp_params* p, const fp_counter_layout* L, const fp_batch* b, const uint8_t* is_dup,
                            fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* counters) {
    if (!p || !L || !b || !out1 || !counters) return FP_E_INVAL;
    if (b->stride > FP_MAX_STRIDE) return FP_E_INVAL;
    if (p->paired && !out2) return FP_E_INVAL;
    ovr_index X;
    if (!ovr_index_make(&X, p, L)) { ovr_index_free(&X); return FP_E_NOMEM; }
    if (p->paired) {
        for (int64_t i = 0; i < b->n; i++)
            process_pe_one(p, &X, L, counters,
                           b->seq1 + i * b->stride, b->qual1 + i * b->stride, b->len1[i],
                           b->seq2 + i * b->stride, b->qual2 + i * b->stride, b->len2[i], is_dup && is_dup[i],
                           out1 + i, out2 + i, ov ? ov + i : NULL);
    } else {
        for (int64_t i = 0; i < b->n; i++)
            process_se_one(p, &X, L, counters, b->seq1 + i * b->stride, b->qual1 + i * b->stride, b->len1[i], is_dup && is_dup[i], out1 + i);
    }
    ovr_index_free(&X);
    return FP_OK;
}

int fp_oracle_process(const fp_params* p, const fp_counter_layout* L, const fp_batch* b,
                      fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* counters) {
    return fp_oracle_process_dedup(p, L, b, NULL, out1, out2, ov, counters);
}

/* Single-function entry points for known-answer tests (tests/test_oracle_kat.py). */
int fp_oracle_trim_and_cut(const fp_params* p, uint8_t* seq, uint8_t* qual, int len, int front, int tail, int* frontOut, int* lenOut) {
    oread r = {seq, qual, len, 0};
    int ft = 0;
    if (!trim_and_cut(p, &r, front, tail, &ft)) return 0;
    *frontOut = (int)(r.seq - seq); *lenOut = r.len;
    return 1;
}
int fp_oracle_trim_polyg(uint8_t* seq, int len, int minLen) { oread r = {seq, seq, len, 0}; trim_polyg(&r, minLen); return r.len; }
int fp_oracle_trim_polyx(uint8_t* seq, int len, int minLen, int* poly, int* plen) {
    oread r = {seq, seq, len, 0}; *poly = 255; *plen = 0; trim_polyx(&r, minLen, poly, plen); return r.len;
}
int fp_oracle_trim_by_sequence(uint8_t* seq, int len, const char* adapter, int* trimmed) {
    int64_t FR[FP_FR_WORDS]; memset(FR, 0, sizeof(FR));
    oread r = {seq, seq, len, 0}; int pos = 0, bases = 0;
    *trimmed = trim_by_sequence(&r, FR, adapter, 4, &pos, &bases);
    return r.len;
}
fp_ov_result fp_oracle_analyze(uint8_t* seq1, int len1, uint8_t* seq2, int len2, int diffLimit, int overlapRequire, double diffPercentLimit) {
    oread r1 = {seq1, seq1, len1, 0}, r2 = {seq2, seq2, len2, 0};
    return analyze(&r1, &r2, diffLimit, overlapRequire, diffPercentLimit, 0);
}
int fp_oracle_pass_filter(const fp_params* p, uint8_t* seq, uint8_t* qual, int len) {
    oread r = {seq, qual, len, 0};
    return pass_filter(p, &r);
}
int fp_oracle_match_with_one_insertion(const uint8_t* insData, const uint8_t* normalData, int cmplen, int diffLimit) {
    return match_with_one_insertion(insData, normalData, cmplen, diffLimit);
}


/* ==========================================================================================
 * FASTQ text <-> rows
 * ========================================================================================== */
/* FastqReader::getLine  src/fastqreader.cpp:240-266 over one in-memory chunk: the line starting at *pos.
 * Returns 0 when no (complete) line is left.  '\n', or '\r' not followed by '\n', ends a line; "\r\n" is one terminator.
 * (The reference's `end < mBufDataLen-1` test leaves the '\n' of a "\r\n" that ends its I/O buffer for the next call, where it
 *  is an empty line that the name search skips -- unobservable, so not restated.) */
static int fq_get_line(const uint8_t* t, int64_t n, int final_chunk, int64_t* pos, int64_t* ls, int64_t* le) {
    int64_t start = *pos, end = start;
    if (start >= n) return 0;
    while (end < n && t[end] != '\r' && t[end] != '\n') end++;                 /* :248-253 */
    if (end >= n && !final_chunk) return 0;                                       /* line not complete in this chunk */
    *ls = start; *le = end;
    if (end < n) {
        end++;                                                                    /* :260 skip \n or \r */
        if (t[end - 1] == '\r' && end < n && t[end] == '\n') end++;               /* :262 handle \r\n */
    }
    *pos = end;
    return 1;
}

int fp_oracle_fastq_decode(const uint8_t* text, int64_t nbytes, int final_chunk, int phred64, int stride,
                           uint8_t* seq, uint8_t* qual, uint16_t* len, int64_t capacity, fp_fastq_rec* recs, fp_fastq_info* info) {
    memset(info, 0, sizeof(*info));
    info->error_record = -1;
    int64_t pos = 0, nrec = 0, nlines = 0;
    /* count lines the way the device reports them (complete lines of the chunk) */
    { int64_t p2 = 0, a, b; while (fq_get_line(text, nbytes, final_chunk, &p2, &a, &b)) nlines++; }
    info->n_lines = nlines;
    for (;;) {
        int64_t save = pos, ns, ne, ss, se, ps, pe, qs, qe;
        /* FastqReader::read :336-343: skip lines until one is non-empty and starts with '@' */
        int got;
        while ((got = fq_get_line(text, nbytes, final_chunk, &pos, &ns, &ne)) && !(ne > ns && text[ns] == '@')) save = pos;
        if (!got) { pos = save; break; }
        if (!fq_get_line(text, nbytes, final_chunk, &pos, &ss, &se) || !fq_get_line(text, nbytes, final_chunk, &pos, &ps, &pe) ||
            !fq_get_line(text, nbytes, final_chunk, &pos, &qs, &qe)) { pos = save; break; }      /* record not complete in this chunk */
        if (nrec >= capacity) { info->more = 1; pos = save; break; }
        int code = FP_FQ_OK;
        if (pe == ps || text[ps] != '+') code = FP_FQ_ERR_STRAND;                 /* :349 */
        else if (qe - qs != se - ss) code = FP_FQ_ERR_LENGTH;                     /* :356 */
        else if (se - ss > stride) code = FP_FQ_ERR_STRIDE;
        if (code != FP_FQ_OK) { info->error = code; info->error_record = nrec; pos = nbytes; break; }   /* the reader returns NULL: input ends */
        const int L = (int)(se - ss);
        uint8_t* srow = seq + (size_t)nrec * stride; uint8_t* qrow = qual + (size_t)nrec * stride;
        memset(srow, 0, stride); memset(qrow, 0, stride);
        memcpy(srow, text + ss, L);
        for (int i = 0; i < L; i++) {
            uint8_t q = text[qs + i];
            if (phred64) { int v = (int)(signed char)q - (64 - 33); q = (uint8_t)(v < 33 ? 33 : v); }   /* read.cpp:35-39 */
            qrow[i] = q;
        }
        len[nrec] = (uint16_t)L;
        recs[nrec].name_off = (uint32_t)ns; recs[nrec].name_len = (uint32_t)(ne - ns);
        recs[nrec].strand_off = (uint32_t)ps; recs[nrec].strand_len = (uint32_t)(pe - ps);
        nrec++;
    }
    info->n_records = nrec;
    info->consumed = pos;
    return 0;
}

/* Read::appendToString  src/read.cpp:119-134 for every read whose pair verdict is PASS and that --dedup did not flag
 * (peprocessor.cpp:575-584, seprocessor.cpp:280-282) */
int64_t fp_oracle_fastq_encode(const uint8_t* text, const fp_fastq_rec* recs, const fp_read_result* res, const uint8_t* seq, const uint8_t* qual,
                               int stride, int64_t n, uint8_t* out, int64_t out_cap) {
    int64_t o = 0;
    for (int64_t i = 0; i < n; i++) {
        if (res[i].pair_verdict != FP_PASS_FILTER || (res[i].flags & FP_F_DUPLICATE)) continue;
        const int64_t need = (int64_t)recs[i].name_len + recs[i].strand_len + 2 * (int64_t)res[i].len + 4;
        if (o + need <= out_cap) {
            uint8_t* d = out + o;
            memcpy(d, text + recs[i].name_off, recs[i].name_len); d += recs[i].name_len; *d++ = '\n';
            memcpy(d, seq + (size_t)i * stride + res[i].front, res[i].len); d += res[i].len; *d++ = '\n';
            memcpy(d, text + recs[i].strand_off, recs[i].strand_len); d += recs[i].strand_len; *d++ = '\n';
            memcpy(d, qual + (size_t)i * stride + res[i].front, res[i].len); d += res[i].len; *d++ = '\n';
        }
        o += need;
    }
    return o;
}


/* ==========================================================================================
 * Duplication bloom filter   src/duplicate.cpp
 * ========================================================================================== */
#include <math.h>
#include <stdlib.h>
#define DUP_PRIME_ARRAY_LEN (1 << 9)                                     /* duplicate.cpp:7 */
struct fp_oracle_dup {
    uint64_t bufLenInBytes, bufLenInBits, offsetMask;
    int bufNum;
    uint8_t* buf;
    uint64_t* primes;
    int64_t total, dups;
};

fp_oracle_dup* fp_oracle_dup_create(int accuracy_level) {                 /* Duplicate::Duplicate :9-66 */
    fp_oracle_dup* d = (fp_oracle_dup*)calloc(1, sizeof(*d));
    d->bufLenInBytes = 1ull << 29; d->bufNum = 2;
    switch (accuracy_level) {
        case 2: d->bufLenInBytes *= 2; break;
        case 3: d->bufLenInBytes *= 2; d->bufNum *= 2; break;
        case 4: d->bufLenInBytes *= 4; d->bufNum *= 2; break;
        case 5: d->bufLenInBytes *= 8; d->bufNum *= 2; break;
        case 6: d->bufLenInBytes *= 8; d->bufNum *= 4; break;
        default: break;
    }
    d->offsetMask = (uint64_t)DUP_PRIME_ARRAY_LEN * d->bufNum - 1;
    d->bufLenInBits = d->bufLenInBytes << 3;
    d->buf = (uint8_t*)calloc(d->bufLenInBytes * d->bufNum, 1);
    d->primes = (uint64_t*)calloc((size_t)d->bufNum * DUP_PRIME_ARRAY_LEN, 8);
    if (!d->buf || !d->primes) { free(d->buf); free(d->primes); free(d); return NULL; }
    uint64_t number = 10000, count = 0;                                   /* initPrimeArrays :68-86 */
    while (count < (uint64_t)d->bufNum * DUP_PRIME_ARRAY_LEN) {
        number++;
        int isPrime = 1;
        for (uint64_t i = 2; i <= sqrt((double)number); i++) if (number % i == 0) { isPrime = 0; break; }
        if (isPrime) { d->primes[count++] = number; number += 10000; }
    }
    return d;
}
void fp_oracle_dup_destroy(fp_oracle_dup* d) { if (d) { free(d->buf); free(d->primes); free(d); } }

static uint64_t dup_hash_val(uint8_t c) {                                 /* SEQ_HASH_VAL :94-112 */
    switch (c) { case 'A': return 7; case 'T': return 222; case 'C': return 74; case 'G': return 31; default: return 13; }
}
static void dup_seq2intvector(const fp_oracle_dup* d, const uint8_t* data, int len, uint64_t* out, int posOffset) {   /* :114-124 */
    for (int p = 0; p < len; p++) {
        const uint64_t base = dup_hash_val(data[p]);
        for (int i = 0; i < d->bufNum; i++) {
            uint64_t offset = (uint64_t)((p + posOffset) * d->bufNum + i) & d->offsetMask;
            out[i] += d->primes[offset] * (base + (uint64_t)(p + posOffset));
        }
    }
}
static int dup_apply(fp_oracle_dup* d, const uint64_t* positions) {       /* applyBloomFilter :156-169 */
    int isDup = 1;
    for (int i = 0; i < d->bufNum; i++) {
        const uint64_t pos = positions[i] % d->bufLenInBits;
        uint8_t* byte = d->buf + (uint64_t)i * d->bufLenInBytes + (pos >> 3);
        const uint8_t bit = (uint8_t)(1u << (pos & 7));
        isDup &= (*byte & bit) != 0;
        *byte |= bit;
    }
    return isDup;
}
void fp_oracle_dup_check(fp_oracle_dup* d, const fp_batch* b, int paired, uint8_t* is_dup) {   /* checkRead :126-139, checkPair :141-154 */
    for (int64_t i = 0; i < b->n; i++) {
        uint64_t positions[8] = {0};
        const int l1 = b->len1[i];
        dup_seq2intvector(d, b->seq1 + (size_t)i * b->stride, l1, positions, 0);
        if (paired) dup_seq2intvector(d, b->seq2 + (size_t)i * b->stride, b->len2[i], positions, l1);
        const int dup = dup_apply(d, positions);
        d->total++; d->dups += dup;
        if (is_dup) is_dup[i] = (uint8_t)dup;
    }
}
void fp_oracle_dup_totals(const fp_oracle_dup* d, int64_t* total, int64_t* dups) { *total = d->total; *dups = d->dups; }
