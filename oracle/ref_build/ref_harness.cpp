// ref_harness.cpp -- drives the REFERENCE's own objects (compiled from /root/reference/src where
// they lie; nothing is copied) over SoA batches and dumps per-read records + private counters in
// the fp_counters layout.  TEST INFRASTRUCTURE (oracle/_ref/libfastp_ref.so): used to pin the C
// port (oracle/fastp_oracle.c), to generate tests/golden fixtures, and as the "reference" CPU
// baseline of bench.py.  Built with -fno-access-control so the private Stats / FilterResult
// counters can be read directly (SURVEY.md App. B).
//
// Every operator below is the reference's function; only the ORDER of calls restates
// SingleEndProcessor::processSingleEnd (src/seprocessor.cpp:204-296) and
// PairEndProcessor::processPairEnd (src/peprocessor.cpp:383-643) + statInsertSize (:710-723),
// because those are private members entangled with reader/writer threads.  The orchestration is
// itself cross-checked against the unmodified CLI (oracle/_ref/fastp_ref) in
// tests/test_reference_cli.py.
#include <string>
#include <mutex>
#include <thread>
#include <vector>
#include <cstring>
#include "options.h"
#include "read.h"
#include "stats.h"
#include "fastqreader.h"
#include "duplicate.h"
#include "evaluator.h"
#include "filter.h"
#include "filterresult.h"
#include "polyx.h"
#include "adaptertrimmer.h"
#include "overlapanalysis.h"
#include "basecorrector.h"
#include "common.h"
#include "fastp_b200.h"

std::string command;          // extern in src/jsonreporter.cpp:21, src/htmlreporter.cpp:6
std::mutex logmtx;            // extern in src/util.h:275

namespace {

void fill_options(Options& o, const fp_params* p) {
    o.trim.front1 = p->trim_front1; o.trim.tail1 = p->trim_tail1;
    o.trim.front2 = p->trim_front2; o.trim.tail2 = p->trim_tail2;
    o.trim.maxLen1 = p->max_len1;   o.trim.maxLen2 = p->max_len2;
    o.qualityCut.enabledFront = p->cut_front; o.qualityCut.enabledTail = p->cut_tail; o.qualityCut.enabledRight = p->cut_right;
    o.qualityCut.windowSizeFront = p->cut_front_window; o.qualityCut.qualityFront = p->cut_front_quality;
    o.qualityCut.windowSizeTail = p->cut_tail_window;   o.qualityCut.qualityTail = p->cut_tail_quality;
    o.qualityCut.windowSizeRight = p->cut_right_window; o.qualityCut.qualityRight = p->cut_right_quality;
    o.polyGTrim.enabled = p->polyg_enabled; o.polyGTrim.minLen = p->polyg_min_len;
    o.polyXTrim.enabled = p->polyx_enabled; o.polyXTrim.minLen = p->polyx_min_len;
    o.adapter.enabled = p->adapter_enabled;
    o.adapter.hasSeqR1 = p->has_seq_r1; o.adapter.hasSeqR2 = p->has_seq_r2;
    o.adapter.sequence = p->adapter_seq_r1 ? p->adapter_seq_r1 : "";
    o.adapter.sequenceR2 = p->adapter_seq_r2 ? p->adapter_seq_r2 : "";
    o.adapter.hasFasta = p->n_fasta_adapters > 0;
    o.adapter.seqsInFasta.clear();
    for (int i = 0; i < p->n_fasta_adapters; i++) o.adapter.seqsInFasta.push_back(p->fasta_adapters[i]);
    o.adapter.allowGapOverlapTrimming = p->allow_gap_overlap_trimming;
    o.adapter.dimerMaxLen = p->dimer_max_len;
    o.correction.enabled = p->correction_enabled;
    o.merge.enabled = p->merge_enabled != 0; o.merge.includeUnmerged = p->merge_include_unmerged != 0;
    o.overlapRequire = p->overlap_require; o.overlapDiffLimit = p->overlap_diff_limit;
    o.overlapDiffPercentLimit = p->overlap_diff_percent_limit;
    o.qualfilter.enabled = p->qual_filter_enabled; o.qualfilter.qualifiedQual = (char)p->qualified_qual;
    o.qualfilter.unqualifiedPercentLimit = p->unqualified_percent_limit;
    o.qualfilter.nBaseLimit = p->n_base_limit; o.qualfilter.avgQualReq = p->avg_qual_req;
    o.lengthFilter.enabled = p->length_filter_enabled; o.lengthFilter.requiredLength = p->length_required;
    o.lengthFilter.maxLength = p->length_limit;
    o.complexityFilter.enabled = p->complexity_filter_enabled; o.complexityFilter.threshold = p->complexity_threshold;
    o.insertSizeMax = p->insert_size_max;
    o.seqLen1 = p->seq_len1; o.seqLen2 = p->seq_len2;
    o.overRepAnalysis.enabled = p->overrep_enabled; o.overRepAnalysis.sampling = p->overrep_sampling;
    o.overRepSeqs1.clear(); o.overRepSeqs2.clear();
    for (int i = 0; i < p->n_overrep1; i++) o.overRepSeqs1[p->overrep_seqs1[i]] = 0;
    for (int i = 0; i < p->n_overrep2; i++) o.overRepSeqs2[p->overrep_seqs2[i]] = 0;
    o.duplicate.enabled = false;
    if (p->paired) { o.in1 = "r1"; o.in2 = "r2"; } else { o.in1 = "r1"; }
}

struct Worker {
    Options opt;
    Filter* filter;
    Stats *pre1, *post1, *pre2, *post2;
    FilterResult* fr;
    std::vector<long> isize;
    Worker(const fp_params* p, int cycles) {
        fill_options(opt, p);
        filter = new Filter(&opt);
        pre1 = new Stats(&opt, false, cycles, 0); post1 = new Stats(&opt, false, cycles, 0);
        pre2 = new Stats(&opt, true, cycles, 0);  post2 = new Stats(&opt, true, cycles, 0);
        fr = new FilterResult(&opt, p->paired);
        isize.assign(p->insert_size_max + 1, 0);
    }
    ~Worker() { delete filter; delete pre1; delete post1; delete pre2; delete post2; delete fr; }
};

Read* make_read(const uint8_t* seq, const uint8_t* qual, int len) {
    return new Read(new std::string("@r"), new std::string((const char*)seq, len), new std::string("+"),
                    new std::string((const char*)qual, len));
}

void fill_result(fp_read_result* o, Read* r, int origLen, int front, int verdict, int pv, int flags,
                 int abases, int polyBase, int polyLen) {
    memset(o, 0, sizeof(*o));
    if (!r) { flags |= FP_F_DROPPED; }
    else { o->front = (uint16_t)front; o->len = (uint16_t)r->length(); }
    (void)origLen;
    o->verdict = (uint8_t)verdict; o->pair_verdict = (uint8_t)pv; o->flags = (uint8_t)flags;
    o->adapter_len = (uint16_t)abases; o->polyx_base = (uint8_t)polyBase; o->polyx_len = (uint16_t)polyLen;
}

// polyX bookkeeping: diff of FilterResult::mTrimmedPolyXReads/Bases around the call
struct PolyXSnap { long reads[4], bases[4]; };
PolyXSnap snap_polyx(FilterResult* fr) { PolyXSnap s; for (int b = 0; b < 4; b++) { s.reads[b] = fr->mTrimmedPolyXReads[b]; s.bases[b] = fr->mTrimmedPolyXBases[b]; } return s; }
bool diff_polyx(FilterResult* fr, const PolyXSnap& s, int& base, int& len) {
    for (int b = 0; b < 4; b++) if (fr->mTrimmedPolyXReads[b] != s.reads[b]) { base = b; len = (int)(fr->mTrimmedPolyXBases[b] - s.bases[b]); return true; }
    return false;
}

void stat_isize(Worker& w, Read* r1, Read* r2, OverlapResult& ov, int ft1, int ft2) {   // peprocessor.cpp:710-723
    int isize = w.opt.insertSizeMax;
    if (ov.overlapped) {
        if (ov.offset > 0) isize = r1->length() + r2->length() - ov.overlap_len + ft1 + ft2;
        else isize = ov.overlap_len + ft1 + ft2;
    }
    if (isize > w.opt.insertSizeMax) isize = w.opt.insertSizeMax;
    w.isize[isize]++;
}

void copy_back(Read* r, int front, uint8_t* seq, uint8_t* qual) {
    // the reference mutates its std::strings; mirror corrected bases into the batch rows
    if (!r) return;
    memcpy(seq + front, r->mSeq->data(), r->length());
    memcpy(qual + front, r->mQuality->data(), r->length());
}

void se_one(Worker& w, const fp_params* p, uint8_t* seq, uint8_t* qual, int len, bool dedupOut, fp_read_result* out) {
    Options* mOptions = &w.opt;
    Read* or1 = make_read(seq, qual, len);
    w.pre1->statRead(or1);                                                    // seprocessor.cpp:211
    int frontTrimmed = 0, flags = dedupOut ? FP_F_DUPLICATE : 0, polyBase = 255, polyLen = 0;
    Read* r1 = w.filter->trimAndCut(or1, mOptions->trim.front1, mOptions->trim.tail1, frontTrimmed);   // :235
    if (r1 != NULL && mOptions->polyGTrim.enabled) {                          // :237-240
        int before = r1->length();
        PolyX::trimPolyG(r1, w.fr, mOptions->polyGTrim.minLen);
        if (r1->length() != before) flags |= FP_F_POLYG_TRIMMED;
    }
    bool isAdapterDimer = false;
    long basesBefore = w.fr->mTrimmedAdapterBases;
    if (r1 != NULL && mOptions->adapter.enabled) {                            // :243-260
        bool trimmed = false;
        if (mOptions->adapter.hasSeqR1) trimmed = AdapterTrimmer::trimBySequence(r1, w.fr, mOptions->adapter.sequence, false);
        if (mOptions->adapter.hasFasta) trimmed |= AdapterTrimmer::trimByMultiSequences(r1, w.fr, mOptions->adapter.seqsInFasta, false);
        if (trimmed) { w.fr->incTrimmedAdapterRead(1); flags |= FP_F_ADAPTER_TRIMMED; }
        if (r1 != NULL && trimmed && r1->length() <= mOptions->adapter.dimerMaxLen) isAdapterDimer = true;
    }
    int abases = (int)(w.fr->mTrimmedAdapterBases - basesBefore);
    if (r1 != NULL && mOptions->polyXTrim.enabled) {                          // :263-266
        PolyXSnap s = snap_polyx(w.fr);
        PolyX::trimPolyX(r1, w.fr, mOptions->polyXTrim.minLen);
        if (diff_polyx(w.fr, s, polyBase, polyLen)) flags |= FP_F_POLYX_TRIMMED;
    }
    if (r1 != NULL) {                                                         // :268-271
        if (mOptions->trim.maxLen1 > 0 && mOptions->trim.maxLen1 < r1->length()) r1->resize(mOptions->trim.maxLen1);
    }
    int result = w.filter->passFilter(r1);                                    // :273
    if (isAdapterDimer) { result = FAIL_ADAPTER_DIMER; flags |= FP_F_ADAPTER_DIMER; }
    w.fr->addFilterResult(result, 1);                                         // :278
    if (!dedupOut && r1 != NULL && result == PASS_FILTER) w.post1->statRead(r1);   // :280-286
    fill_result(out, r1, len, frontTrimmed, result, result, flags, abases, polyBase, polyLen);
    (void)p;
    delete or1;   // r1 == or1 or NULL (trimAndCut mutates in place)
}

void pe_one(Worker& w, const fp_params* p, uint8_t* seq1, uint8_t* qual1, int len1, uint8_t* seq2, uint8_t* qual2, int len2, bool dedupOut,
            fp_read_result* out1, fp_read_result* out2, fp_ov_result* ovOut) {
    Options* mOptions = &w.opt;
    const bool tid0 = p->thread0_semantics != 0;
    Read* or1 = make_read(seq1, qual1, len1);
    Read* or2 = make_read(seq2, qual2, len2);
    w.pre1->statRead(or1);                                                    // peprocessor.cpp:393-394
    w.pre2->statRead(or2);
    int frontTrimmed1 = 0, frontTrimmed2 = 0;
    int flags1 = dedupOut ? FP_F_DUPLICATE : 0, flags2 = flags1, pb1 = 255, pb2 = 255, pl1 = 0, pl2 = 0, ab1 = 0, ab2 = 0;   // :397-401
    Read* r1 = w.filter->trimAndCut(or1, mOptions->trim.front1, mOptions->trim.tail1, frontTrimmed1);   // :425-426
    Read* r2 = w.filter->trimAndCut(or2, mOptions->trim.front2, mOptions->trim.tail2, frontTrimmed2);
    if (r1 != NULL && r2 != NULL && mOptions->polyGTrim.enabled) {            // :428-431
        int b1 = r1->length(), b2 = r2->length();
        PolyX::trimPolyG(r1, r2, w.fr, mOptions->polyGTrim.minLen);
        if (r1->length() != b1) flags1 |= FP_F_POLYG_TRIMMED;
        if (r2->length() != b2) flags2 |= FP_F_POLYG_TRIMMED;
    }
    bool isizeEvaluated = false, isAdapterDimer = false;
    OverlapResult ov = {};
    bool ovComputed = false;
    if (r1 != NULL && r2 != NULL && (mOptions->adapter.enabled || mOptions->correction.enabled || tid0 || mOptions->merge.enabled)) {   // :438-441
        ov = OverlapAnalysis::analyze(r1, r2, mOptions->overlapDiffLimit, mOptions->overlapRequire, mOptions->overlapDiffPercentLimit / 100.0);
        ovComputed = true;
    }
    if (r1 != NULL && r2 != NULL && (mOptions->adapter.enabled || mOptions->correction.enabled)) {   // :443
        OverlapResult ovForAdapter = mOptions->adapter.allowGapOverlapTrimming                                             // :445-447
            ? OverlapAnalysis::analyze(r1, r2, mOptions->overlapDiffLimit, mOptions->overlapRequire, mOptions->overlapDiffPercentLimit / 100.0, true) : ov;
        if (tid0) { stat_isize(w, r1, r2, ov, frontTrimmed1, frontTrimmed2); isizeEvaluated = true; }   // :449-452
        if (mOptions->correction.enabled && !ovForAdapter.hasGap) {           // :453-456
            std::string s1 = *r1->mSeq, s2 = *r2->mSeq;
            BaseCorrector::correctByOverlapAnalysis(r1, r2, w.fr, ovForAdapter);
            if (s1 != *r1->mSeq) flags1 |= FP_F_CORRECTED;
            if (s2 != *r2->mSeq) flags2 |= FP_F_CORRECTED;
            copy_back(r1, frontTrimmed1, seq1, qual1);
            copy_back(r2, frontTrimmed2, seq2, qual2);
        }
        if (mOptions->adapter.enabled) {                                      // :457-485
            int l1 = r1->length(), l2 = r2->length();
            long basesBefore = w.fr->mTrimmedAdapterBases;
            bool trimmed = AdapterTrimmer::trimByOverlapAnalysis(r1, r2, w.fr, ovForAdapter, frontTrimmed1, frontTrimmed2);
            if (trimmed) { ab1 += l1 - r1->length(); ab2 += l2 - r2->length(); }
            bool trimmed1 = trimmed, trimmed2 = trimmed;
            if (!trimmed) {
                if (mOptions->adapter.hasSeqR1) {
                    long b = w.fr->mTrimmedAdapterBases;
                    trimmed1 = AdapterTrimmer::trimBySequence(r1, w.fr, mOptions->adapter.sequence, false);
                    ab1 += (int)(w.fr->mTrimmedAdapterBases - b);
                }
                if (mOptions->adapter.hasSeqR2) {
                    long b = w.fr->mTrimmedAdapterBases;
                    trimmed2 = AdapterTrimmer::trimBySequence(r2, w.fr, mOptions->adapter.sequenceR2, true);
                    ab2 += (int)(w.fr->mTrimmedAdapterBases - b);
                }
            }
            if (mOptions->adapter.hasFasta) {
                long b = w.fr->mTrimmedAdapterBases;
                trimmed1 |= AdapterTrimmer::trimByMultiSequences(r1, w.fr, mOptions->adapter.seqsInFasta, false);
                ab1 += (int)(w.fr->mTrimmedAdapterBases - b);
                b = w.fr->mTrimmedAdapterBases;
                trimmed2 |= AdapterTrimmer::trimByMultiSequences(r2, w.fr, mOptions->adapter.seqsInFasta, true);
                ab2 += (int)(w.fr->mTrimmedAdapterBases - b);
            }
            (void)basesBefore;
            if (trimmed1) { w.fr->incTrimmedAdapterRead(1); flags1 |= FP_F_ADAPTER_TRIMMED; }
            if (trimmed2) { w.fr->incTrimmedAdapterRead(1); flags2 |= FP_F_ADAPTER_TRIMMED; }
            if (r1 != NULL && r2 != NULL && (trimmed1 || trimmed2) &&
                r1->length() <= mOptions->adapter.dimerMaxLen && r2->length() <= mOptions->adapter.dimerMaxLen)
                isAdapterDimer = true;
        }
    }
    if (tid0 && !isizeEvaluated && r1 != NULL && r2 != NULL) {                // :497-504
        if (!ovComputed) {
            ov = OverlapAnalysis::analyze(r1, r2, mOptions->overlapDiffLimit, mOptions->overlapRequire, mOptions->overlapDiffPercentLimit / 100.0);
            ovComputed = true;
        }
        stat_isize(w, r1, r2, ov, frontTrimmed1, frontTrimmed2);
        isizeEvaluated = true;
    }
    if (r1 != NULL && r2 != NULL && mOptions->polyXTrim.enabled) {            // :506-509
        PolyXSnap s = snap_polyx(w.fr);
        PolyX::trimPolyX(r1, w.fr, mOptions->polyXTrim.minLen);
        if (diff_polyx(w.fr, s, pb1, pl1)) flags1 |= FP_F_POLYX_TRIMMED;
        s = snap_polyx(w.fr);
        PolyX::trimPolyX(r2, w.fr, mOptions->polyXTrim.minLen);
        if (diff_polyx(w.fr, s, pb2, pl2)) flags2 |= FP_F_POLYX_TRIMMED;
    }
    if (r1 != NULL && r2 != NULL) {                                           // :511-516
        if (mOptions->trim.maxLen1 > 0 && mOptions->trim.maxLen1 < r1->length()) r1->resize(mOptions->trim.maxLen1);
        if (mOptions->trim.maxLen2 > 0 && mOptions->trim.maxLen2 < r2->length()) r2->resize(mOptions->trim.maxLen2);
    }
    int result1 = 0, result2 = 0, pv = 0;
    bool mergeProcessed = false;
    if (mOptions->merge.enabled && r1 && r2) {                                // :519-560
        ov = OverlapAnalysis::analyze(r1, r2, mOptions->overlapDiffLimit, mOptions->overlapRequire, mOptions->overlapDiffPercentLimit / 100.0);
        ovComputed = true;
        if (ov.overlapped) {
            Read* merged = OverlapAnalysis::merge(r1, r2, ov);
            int result = w.filter->passFilter(merged);
            w.fr->addFilterResult(result, 2);
            if (result == PASS_FILTER) { w.post1->statRead(merged); w.fr->addMergedPairs(1); }
            delete merged;
            result1 = result2 = pv = result;
            flags1 |= FP_F_MERGED; flags2 |= FP_F_MERGED;
            mergeProcessed = true;
        } else if (mOptions->merge.includeUnmerged) {
            result1 = w.filter->passFilter(r1);
            result2 = w.filter->passFilter(r2);
            if (isAdapterDimer) { result1 = FAIL_ADAPTER_DIMER; result2 = FAIL_ADAPTER_DIMER; flags1 |= FP_F_ADAPTER_DIMER; flags2 |= FP_F_ADAPTER_DIMER; }
            w.fr->addFilterResult(result1, 1);
            if (result1 == PASS_FILTER && !dedupOut) w.post1->statRead(r1);   // :547
            w.fr->addFilterResult(result2, 1);
            if (result2 == PASS_FILTER && !dedupOut) w.post1->statRead(r2);   // :553
            pv = std::max(result1, result2);
            mergeProcessed = true;
        }
    }
    if (!mergeProcessed) {
        result1 = w.filter->passFilter(r1);                                   // :565-566
        result2 = w.filter->passFilter(r2);
        if (isAdapterDimer) { result1 = FAIL_ADAPTER_DIMER; result2 = FAIL_ADAPTER_DIMER; flags1 |= FP_F_ADAPTER_DIMER; flags2 |= FP_F_ADAPTER_DIMER; }
        pv = std::max(result1, result2);
        w.fr->addFilterResult(pv, 2);                                         // :573
        if (!dedupOut && !mOptions->merge.enabled && r1 != NULL && result1 == PASS_FILTER && r2 != NULL && result2 == PASS_FILTER) {   // :575-591
            w.post1->statRead(r1);
            w.post2->statRead(r2);
        }
    }
    fill_result(out1, r1, len1, frontTrimmed1, result1, pv, flags1, ab1, pb1, pl1);
    fill_result(out2, r2, len2, frontTrimmed2, result2, pv, flags2, ab2, pb2, pl2);
    if (ovOut) {
        ovOut->overlapped = ov.overlapped; ovOut->has_gap = ov.hasGap;
        ovOut->offset = (int16_t)ov.offset; ovOut->overlap_len = (int16_t)ov.overlap_len; ovOut->diff = (int16_t)ov.diff;
    }
    delete or1; delete or2;
}

void dump_stats(Stats* s, const fp_params* p, const fp_counter_layout* L, int idx, int64_t* C) {
    int n = std::min(s->mBufLen, L->cycles);
    for (int k = 0; k < 8; k++)
        for (int c = 0; c < n; c++) {
            C[fp_off_cycle(L, idx, 0 * 8 + k, c)] += s->mCycleQ30Bases[k][c];
            C[fp_off_cycle(L, idx, 1 * 8 + k, c)] += s->mCycleQ20Bases[k][c];
            C[fp_off_cycle(L, idx, 2 * 8 + k, c)] += s->mCycleBaseContents[k][c];
            C[fp_off_cycle(L, idx, 3 * 8 + k, c)] += s->mCycleBaseQual[k][c];
        }
    for (int c = 0; c < n; c++) {
        C[fp_off_cycle(L, idx, 32, c)] += s->mCycleTotalBase[c];
        C[fp_off_cycle(L, idx, 33, c)] += s->mCycleTotalQual[c];
    }
    for (int k = 0; k < FP_KMER_BINS; k++) C[fp_off_kmer(L, idx, k)] += s->mKmer[k];
    for (int q = 0; q < FP_QUAL_BINS; q++) C[fp_off_qualhist(L, idx, q)] += s->mBaseQualHistogram[q];
    C[fp_off_reads(L, idx)] += s->mReads;
    C[fp_off_length_sum(L, idx)] += s->mLengthSum;
    if (p->overrep_enabled) {                                                 // Stats::mOverRepSeq / mOverRepSeqDist (stats.h:91-92)
        const int side = idx >> 1;
        const char* const* cands = side ? p->overrep_seqs2 : p->overrep_seqs1;
        for (int k = 0; k < L->n_overrep[side]; k++) {
            std::string key(cands[k]);
            if (s->mOverRepSeq.count(key) == 0) continue;
            C[fp_off_overrep_count(L, idx, k)] += s->mOverRepSeq[key];
            long* dist = s->mOverRepSeqDist[key];
            for (int q = 0; q < L->overrep_len[side] && q < s->mEvaluatedSeqLen; q++) C[fp_off_overrep_dist(L, idx, k, q)] += dist[q];
        }
    }
}

void dump_worker(Worker& w, const fp_params* p, const fp_counter_layout* L, int64_t* C) {
    dump_stats(w.pre1, p, L, FP_STATS_PRE1, C);
    dump_stats(w.post1, p, L, FP_STATS_POST1, C);
    if (p->paired) { dump_stats(w.pre2, p, L, FP_STATS_PRE2, C); dump_stats(w.post2, p, L, FP_STATS_POST2, C); }
    int64_t* FR = C + L->off_filter;
    for (int i = 0; i < FILTER_RESULT_TYPES; i++) FR[FP_FR_READSTATS + i] += w.fr->mFilterReadStats[i];
    FR[FP_FR_ADAPTER_READS] += w.fr->mTrimmedAdapterRead;
    FR[FP_FR_ADAPTER_BASES] += w.fr->mTrimmedAdapterBases;
    for (int b = 0; b < 4; b++) { FR[FP_FR_POLYX_READS + b] += w.fr->mTrimmedPolyXReads[b]; FR[FP_FR_POLYX_BASES + b] += w.fr->mTrimmedPolyXBases[b]; }
    for (int i = 0; i < 64; i++) FR[FP_FR_CORRECTION + i] += w.fr->mCorrectionMatrix[i];
    FR[FP_FR_CORRECTED_READS] += w.fr->mCorrectedReads;
    FR[FP_FR_MERGED_PAIRS] += w.fr->mMergedPairs;
    for (int i = 0; i < L->isize_bins && i < (int)w.isize.size(); i++) C[L->off_isize + i] += w.isize[i];
}

void run_range(const fp_params* p, const fp_counter_layout* L, const fp_batch* b, int64_t lo, int64_t hi,
               fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* C, const uint8_t* is_dup = nullptr) {
    Worker w(p, L->cycles);
    fp_read_result tmp1, tmp2;
    for (int64_t i = lo; i < hi; i++) {
        if (p->paired)
            pe_one(w, p, b->seq1 + i * b->stride, b->qual1 + i * b->stride, b->len1[i],
                   b->seq2 + i * b->stride, b->qual2 + i * b->stride, b->len2[i], is_dup && is_dup[i],
                   out1 ? out1 + i : &tmp1, out2 ? out2 + i : &tmp2, ov ? ov + i : NULL);
        else
            se_one(w, p, b->seq1 + i * b->stride, b->qual1 + i * b->stride, b->len1[i], is_dup && is_dup[i], out1 ? out1 + i : &tmp1);
    }
    dump_worker(w, p, L, C);
}

}  // namespace

extern "C" {

// Same contract as fp_oracle_process (oracle/fastp_oracle.h). Counters are ADDED into `counters`.
int fp_ref_process(const fp_params* p, const fp_counter_layout* L, const fp_batch* b,
                   fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* counters) {
    run_range(p, L, b, 0, b->n, out1, out2, ov, counters);
    return FP_OK;
}

// Same contract as fp_oracle_process_dedup: is_dup[i] is what `mDuplicate->checkPair(or1, or2) && mOptions->duplicate.dedup` gave for unit i.
int fp_ref_process_dedup(const fp_params* p, const fp_counter_layout* L, const fp_batch* b, const uint8_t* is_dup,
                         fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* counters) {
    run_range(p, L, b, 0, b->n, out1, out2, ov, counters, is_dup);
    return FP_OK;
}

// Single worker over the whole batch + the reference's own adapter-string histograms (FilterResult::mAdapter1 / mAdapter2,
// src/filterresult.cpp:124-180) serialised as "1\tSEQ\tCOUNT\n" / "2\t..." lines in map order.  Returns the number of lines.
int fp_ref_process_maps(const fp_params* p, const fp_counter_layout* L, const fp_batch* b, int64_t* counters, char* out, int64_t cap, int64_t* used) {
    Worker w(p, L->cycles);
    fp_read_result t1, t2;
    for (int64_t i = 0; i < b->n; i++) {
        if (p->paired)
            pe_one(w, p, b->seq1 + i * b->stride, b->qual1 + i * b->stride, b->len1[i], b->seq2 + i * b->stride, b->qual2 + i * b->stride, b->len2[i], false, &t1, &t2, NULL);
        else
            se_one(w, p, b->seq1 + i * b->stride, b->qual1 + i * b->stride, b->len1[i], false, &t1);
    }
    dump_worker(w, p, L, counters);
    std::string o; int n = 0;
    for (auto& kv : w.fr->mAdapter1) { o += "1\t" + kv.first + "\t" + std::to_string(kv.second) + "\n"; n++; }
    for (auto& kv : w.fr->mAdapter2) { o += "2\t" + kv.first + "\t" + std::to_string(kv.second) + "\n"; n++; }
    *used = (int64_t)o.size();
    if ((int64_t)o.size() <= cap) memcpy(out, o.data(), o.size());
    return n;
}

// Multi-threaded form for the CPU baseline: `nthreads` workers over contiguous ranges, private
// Stats/FilterResult per worker, summed at the end (what Stats::merge / FilterResult::merge do).
// out1/out2/ov may be NULL (baseline timing).
int fp_ref_process_mt(const fp_params* p, const fp_counter_layout* L, const fp_batch* b,
                      fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov, int64_t* counters, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    std::vector<std::vector<int64_t>> part(nthreads, std::vector<int64_t>(L->total, 0));
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; t++) {
        int64_t lo = b->n * t / nthreads, hi = b->n * (t + 1) / nthreads;
        th.emplace_back([=, &part]() { run_range(p, L, b, lo, hi, out1, out2, ov, part[t].data()); });
    }
    for (auto& x : th) x.join();
    for (int t = 0; t < nthreads; t++)
        for (int64_t i = 0; i < L->total; i++) counters[i] += part[t][i];
    return FP_OK;
}

// FastqReader itself (src/fastqreader.cpp) over a plain FASTQ file: every record it returns, flattened as
// [name_len, seq_len, strand_len, qual_len] (4 x int32) followed by the four byte strings.  Returns the record count,
// *used = bytes written (nothing is written past cap, the count still runs on).
int64_t fp_ref_fastq_read_file(const char* path, int phred64, uint8_t* out, int64_t cap, int64_t* used) {
    FastqReader reader(path, true, phred64 != 0);
    int64_t n = 0, o = 0;
    for (;;) {
        Read* r = reader.read();
        if (!r) break;
        const std::string* f[4] = {r->mName, r->mSeq, r->mStrand, r->mQuality};
        int64_t need = 16;
        for (int k = 0; k < 4; k++) need += (int64_t)f[k]->size();
        if (o + need <= cap) {
            int32_t* h = reinterpret_cast<int32_t*>(out + o);
            for (int k = 0; k < 4; k++) h[k] = (int32_t)f[k]->size();
            uint8_t* d = out + o + 16;
            for (int k = 0; k < 4; k++) { memcpy(d, f[k]->data(), f[k]->size()); d += f[k]->size(); }
        }
        o += need;
        n++;
        delete r;
    }
    *used = o;
    return n;
}

// The reference's own Evaluator::computeOverRepSeq (src/evaluator.cpp:78-169) over a plain FASTQ file: the candidate
// sequences NUL-separated in map order; returns how many (*used = bytes needed).
int fp_ref_compute_overrep(const char* path, int seqlen, char* out, int64_t cap, int64_t* used) {
    Options opt;
    Evaluator ev(&opt);
    std::map<std::string, long> hot;
    ev.computeOverRepSeq(path, hot, seqlen);
    int64_t o = 0; int n = 0;
    for (auto& kv : hot) {
        const int64_t need = (int64_t)kv.first.size() + 1;
        if (o + need <= cap) memcpy(out + o, kv.first.c_str(), (size_t)need);
        o += need; n++;
    }
    *used = o;
    return n;
}

// The reference's own Duplicate object (src/duplicate.cpp), units fed in index order.
struct fp_ref_dup { Options opt; Duplicate* d; int64_t total = 0, dups = 0; };
void* fp_ref_dup_create(int accuracy_level) {
    fp_ref_dup* h = new fp_ref_dup();
    h->opt.duplicate.enabled = true; h->opt.duplicate.accuracyLevel = accuracy_level;
    h->d = new Duplicate(&h->opt);
    return h;
}
void fp_ref_dup_destroy(void* hp) { fp_ref_dup* h = (fp_ref_dup*)hp; delete h->d; delete h; }
void fp_ref_dup_check(void* hp, const fp_batch* b, int paired, uint8_t* is_dup) {
    fp_ref_dup* h = (fp_ref_dup*)hp;
    for (int64_t i = 0; i < b->n; i++) {
        Read r1("@a", std::string((const char*)b->seq1 + (size_t)i * b->stride, b->len1[i]).c_str(), "+", std::string(b->len1[i], 'I').c_str());
        bool dup;
        if (paired) {
            Read r2("@a", std::string((const char*)b->seq2 + (size_t)i * b->stride, b->len2[i]).c_str(), "+", std::string(b->len2[i], 'I').c_str());
            dup = h->d->checkPair(&r1, &r2);
        } else dup = h->d->checkRead(&r1);
        h->total++; h->dups += dup ? 1 : 0;
        if (is_dup) is_dup[i] = dup ? 1 : 0;
    }
}
void fp_ref_dup_totals(void* hp, int64_t* total, int64_t* dups, double* rate) {
    fp_ref_dup* h = (fp_ref_dup*)hp; *total = h->total; *dups = h->dups; *rate = h->d->getDupRate();
}

}  // extern "C"
