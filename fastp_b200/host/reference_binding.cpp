/*
 * reference_binding.cpp -- the binding a fastp maintainer adds: the two worker bodies
 *     bool SingleEndProcessor::processSingleEnd(ReadPack*, ThreadConfig*)      src/seprocessor.cpp:197-325
 *     bool PairEndProcessor::processPairEnd(ReadPack*, ReadPack*, ThreadConfig*) src/peprocessor.cpp:362-708
 * re-implemented on top of libfastp_b200.so, compiled against the REFERENCE'S OWN HEADERS (this file is useless without them).
 *
 * How it is built (oracle/Makefile, target _ref/fastp_gpu): the reference's sources are compiled where they lie; in private copies of
 * peprocessor.{h,cpp} / seprocessor.{h,cpp} under oracle/_ref/patched the two member functions are RENAMED by sed to
 * processPairEnd_cpu / processSingleEnd_cpu (one declaration added per class), nothing else is touched; this file then supplies
 * the functions under their original names.  Everything around them -- CLI, Evaluator, reader / writer threads, pack queues,
 * duplicate filter, Stats::merge, the JSON / HTML reporters -- is the unmodified reference.
 *
 * Per pack:  host-only pre-steps in the reference's order (duplicate check, index filter, MGI fix)  ->  stage the Read strings into
 * pinned SoA rows  ->  fp_process_*_host (the whole operator chain on the device)  ->  unstage: apply trim windows and corrected
 * bases to the Read objects, replay the adapter-string events through the reference's own FilterResult::addAdapterTrimmed, add the
 * device's counter block to this worker's Stats / FilterResult objects, then the unchanged tail of the reference loop (output
 * strings, writers, recycling).  Merging mode (--merge / --include_unmerged, :519-560) runs on the device too: the merged Read is built
 * by the reference's own OverlapAnalysis::merge from the device's second overlap record.  Option sets the device path does not
 * cover (overlapped_out, UMI, over-representation analysis, reads longer than FP_MAX_STRIDE, adapters past fp_ctx_create's limits) are
 * handed to the stock body.
 */
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "peprocessor.h"
#include "seprocessor.h"
#include "adaptertrimmer.h"
#include "duplicate.h"
#include "filter.h"
#include "filterresult.h"
#include "overlapanalysis.h"
/* Stats::extendBuffer (private) is called below before the block of merged reads -- up to two reads long -- is added to the post-filter
   Stats; this file is built with -fno-access-control (oracle/Makefile).  A maintainer would rather add the block-adding function to Stats. */
#include "stats.h"
#include "threadconfig.h"
#include "umiprocessor.h"
#include "writerthread.h"
#include "fastp_b200.h"

namespace {

struct GpuWorker {                    /* one per worker thread (ThreadConfig), like the reference's per-thread Stats */
    fp_ctx* ctx = nullptr;
    fp_params params;
    fp_counter_layout L;
    int stride = 0;
    int64_t cap = 0;
    uint8_t *seq[2] = {nullptr, nullptr}, *qual[2] = {nullptr, nullptr};
    uint16_t* len[2] = {nullptr, nullptr};
    fp_read_result* res[2] = {nullptr, nullptr};
    fp_ov_result* ov = nullptr;
    std::vector<fp_patch> patches;
    std::vector<fp_adapter_event> events;
    std::vector<int64_t> block;
    std::vector<const char*> fastaKeep;
    std::vector<std::string> adapters;    /* 0 = sequence, 1 = sequenceR2, 2+i = seqsInFasta[i] */
    long packs = 0;
};

std::mutex g_mu;
std::map<std::pair<const void*, int>, GpuWorker*> g_workers;

void die(const char* what) {
    fprintf(stderr, "fastp_b200 binding: %s: %s\n", what, fp_last_error());
    exit(-1);                          /* error_exit() style: the reference aborts on fatal errors too (src/util.h) */
}

void fill_params(fp_params* p, Options* o, bool paired, int tid, GpuWorker* w) {
    fp_params_default(p, paired ? 1 : 0);
    p->thread0_semantics = tid == 0 ? 1 : 0;                                   /* src/peprocessor.cpp:438,449,497 */
    p->trim_front1 = o->trim.front1; p->trim_tail1 = o->trim.tail1; p->trim_front2 = o->trim.front2; p->trim_tail2 = o->trim.tail2;
    p->max_len1 = o->trim.maxLen1; p->max_len2 = o->trim.maxLen2;
    p->cut_front = o->qualityCut.enabledFront; p->cut_tail = o->qualityCut.enabledTail; p->cut_right = o->qualityCut.enabledRight;
    p->cut_front_window = o->qualityCut.windowSizeFront; p->cut_front_quality = o->qualityCut.qualityFront;
    p->cut_tail_window = o->qualityCut.windowSizeTail; p->cut_tail_quality = o->qualityCut.qualityTail;
    p->cut_right_window = o->qualityCut.windowSizeRight; p->cut_right_quality = o->qualityCut.qualityRight;
    p->polyg_enabled = o->polyGTrim.enabled; p->polyg_min_len = o->polyGTrim.minLen;
    p->polyx_enabled = o->polyXTrim.enabled; p->polyx_min_len = o->polyXTrim.minLen;
    p->adapter_enabled = o->adapter.enabled; p->has_seq_r1 = o->adapter.hasSeqR1; p->has_seq_r2 = o->adapter.hasSeqR2;
    p->adapter_seq_r1 = o->adapter.sequence.c_str(); p->adapter_seq_r2 = o->adapter.sequenceR2.c_str();
    w->fastaKeep.clear();
    if (o->adapter.hasFasta) for (auto& s : o->adapter.seqsInFasta) w->fastaKeep.push_back(s.c_str());
    p->n_fasta_adapters = (int)w->fastaKeep.size(); p->fasta_adapters = w->fastaKeep.empty() ? nullptr : w->fastaKeep.data();
    p->allow_gap_overlap_trimming = o->adapter.allowGapOverlapTrimming; p->dimer_max_len = o->adapter.dimerMaxLen;
    p->correction_enabled = o->correction.enabled;
    p->overlap_require = o->overlapRequire; p->overlap_diff_limit = o->overlapDiffLimit; p->overlap_diff_percent_limit = o->overlapDiffPercentLimit;
    p->qual_filter_enabled = o->qualfilter.enabled; p->qualified_qual = (unsigned char)o->qualfilter.qualifiedQual;
    p->unqualified_percent_limit = o->qualfilter.unqualifiedPercentLimit; p->n_base_limit = o->qualfilter.nBaseLimit; p->avg_qual_req = o->qualfilter.avgQualReq;
    p->length_filter_enabled = o->lengthFilter.enabled; p->length_required = o->lengthFilter.requiredLength; p->length_limit = o->lengthFilter.maxLength;
    p->complexity_filter_enabled = o->complexityFilter.enabled; p->complexity_threshold = o->complexityFilter.threshold;
    p->insert_size_max = o->insertSizeMax; p->seq_len1 = o->seqLen1; p->seq_len2 = o->seqLen2;
    p->overrep_enabled = 0;
    p->merge_enabled = paired && o->merge.enabled; p->merge_include_unmerged = o->merge.includeUnmerged;
    w->adapters.clear();
    w->adapters.push_back(o->adapter.sequence); w->adapters.push_back(o->adapter.sequenceR2);
    for (auto& s : o->adapter.seqsInFasta) w->adapters.push_back(s);
}

GpuWorker* worker_for(const void* proc, Options* o, bool paired, int tid, int need_len, int64_t need_cap) {
    std::lock_guard<std::mutex> lk(g_mu);
    GpuWorker*& w = g_workers[{proc, tid}];
    if (w && (need_len > w->stride || need_cap > w->cap)) {                    /* a longer read / larger pack than planned for: rebuild */
        return nullptr;
    }
    if (w) return w;
    w = new GpuWorker();
    fill_params(&w->params, o, paired, tid, w);
    const int want = std::max(need_len, std::max(o->seqLen1, o->seqLen2)) + 8;
    w->stride = std::min(FP_MAX_STRIDE, std::max(32, (want + 15) / 16 * 16));
    if (paired && w->stride > 256) w->stride = 256;                            /* the column pass covers 2 x 256 cycles (fp_ctx_create) */
    w->cap = std::max<int64_t>(need_cap, 4096);
    const char* dev = getenv("FASTP_B200_DEVICE");
    /* merged reads are up to two rows long: the counter block covers 2 x stride cycles then */
    if (fp_ctx_create(&w->params, dev ? atoi(dev) : 0, w->cap, w->stride, w->params.merge_enabled ? 2 * w->stride : w->stride, &w->ctx) != FP_OK) die("fp_ctx_create");
    fp_ctx_layout(w->ctx, &w->L);
    w->block.resize(w->L.total);
    const int sides = paired ? 2 : 1;
    for (int s = 0; s < sides; s++) {
        if (fp_host_alloc((void**)&w->seq[s], (size_t)w->cap * w->stride) || fp_host_alloc((void**)&w->qual[s], (size_t)w->cap * w->stride) ||
            fp_host_alloc((void**)&w->len[s], (size_t)w->cap * 2) || fp_host_alloc((void**)&w->res[s], (size_t)w->cap * sizeof(fp_read_result)))
            die("fp_host_alloc");
    }
    if (paired && fp_host_alloc((void**)&w->ov, (size_t)w->cap * sizeof(fp_ov_result))) die("fp_host_alloc");
    w->patches.resize((size_t)w->cap * 8 + 1024);
    w->events.resize((size_t)w->cap * (4 + 2 * w->fastaKeep.size()) + 1024);
    return w;
}

/* fp_ctx_create refuses adapters longer than FP_MAX_ADAPTER_LEN and more than FP_MAX_ADAPTERS fasta entries; the reference's loader
   keeps both (src/options.cpp loadFastaAdapters drops only entries under 6 bases and duplicates), so such option sets run on the stock body */
bool adapters_fit(Options* o) {
    if ((o->adapter.hasSeqR1 && o->adapter.sequence.size() > FP_MAX_ADAPTER_LEN) || (o->adapter.hasSeqR2 && o->adapter.sequenceR2.size() > FP_MAX_ADAPTER_LEN))
        return false;
    if (!o->adapter.hasFasta) return true;
    if (o->adapter.seqsInFasta.size() > FP_MAX_ADAPTERS) return false;
    for (auto& s : o->adapter.seqsInFasta) if (s.size() > FP_MAX_ADAPTER_LEN) return false;
    return true;
}

bool supported(Options* o, bool hasOverlappedWriter) {
    return !hasOverlappedWriter && !o->umi.enabled && !o->overRepAnalysis.enabled && adapters_fit(o);
}

void stage(GpuWorker* w, int side, int64_t i, Read* r) {
    const int n = r->length();
    memcpy(w->seq[side] + i * w->stride, r->mSeq->data(), n);
    memcpy(w->qual[side] + i * w->stride, r->mQuality->data(), n);
    w->len[side][i] = (uint16_t)n;
}

/* Filter::trimAndCut / resize as the reference's in-place string edits (src/filter.cpp:196-206): returns NULL for a dropped read */
Read* unstage(GpuWorker* w, int side, int64_t i, Read* r) {
    const fp_read_result& x = w->res[side][i];
    if (x.flags & FP_F_DROPPED) return NULL;
    if (x.flags & FP_F_CORRECTED) {                                            /* BaseCorrector rewrote bases in place */
        r->mSeq->assign((const char*)w->seq[side] + i * w->stride, r->mSeq->size());
        r->mQuality->assign((const char*)w->qual[side] + i * w->stride, r->mQuality->size());
    }
    if (x.front) { r->mSeq->erase(0, x.front); r->mQuality->erase(0, x.front); }
    r->mSeq->resize(x.len); r->mQuality->resize(x.len);
    return r;
}

/* add the device's counter block to this worker's Stats / FilterResult (what statRead / addFilterResult / addPolyXTrimmed ...
 * would have accumulated), then clear it on the device */
void add_stats(Stats* s, const int64_t* B, const fp_counter_layout& L, int which) {
    int used = 0;                                                              /* cycles the block really holds (merged reads: beyond the buffer) */
    for (int c = 0; c < (int)L.cycles; c++) if (B[fp_off_cycle(&L, which, 32, c)]) used = c + 1;
    if (used > s->mBufLen) s->extendBuffer(std::max(used + 100, (int)(used * 1.5)));   /* what statRead does for a longer read (stats.cpp:195-197) */
    const int n = std::min(s->mBufLen, (int)L.cycles);
    for (int b = 0; b < 8; b++)
        for (int c = 0; c < n; c++) {
            s->mCycleQ30Bases[b][c] += B[fp_off_cycle(&L, which, 0 * 8 + b, c)];
            s->mCycleQ20Bases[b][c] += B[fp_off_cycle(&L, which, 1 * 8 + b, c)];
            s->mCycleBaseContents[b][c] += B[fp_off_cycle(&L, which, 2 * 8 + b, c)];
            s->mCycleBaseQual[b][c] += B[fp_off_cycle(&L, which, 3 * 8 + b, c)];
        }
    for (int c = 0; c < n; c++) { s->mCycleTotalBase[c] += B[fp_off_cycle(&L, which, 32, c)]; s->mCycleTotalQual[c] += B[fp_off_cycle(&L, which, 33, c)]; }
    for (int k = 0; k < FP_KMER_BINS; k++) s->mKmer[k] += B[fp_off_kmer(&L, which, k)];
    for (int q = 0; q < FP_QUAL_BINS; q++) s->mBaseQualHistogram[q] += B[fp_off_qualhist(&L, which, q)];
    s->mReads += B[fp_off_reads(&L, which)];
    s->mLengthSum += B[fp_off_length_sum(&L, which)];
}

void add_counters(GpuWorker* w, ThreadConfig* config, bool paired, std::atomic_long* isize) {
    if (fp_counters_fetch(w->ctx, w->block.data()) != FP_OK) die("fp_counters_fetch");
    const int64_t* B = w->block.data();
    add_stats(config->getPreStats1(), B, w->L, FP_STATS_PRE1);
    add_stats(config->getPostStats1(), B, w->L, FP_STATS_POST1);
    if (paired) { add_stats(config->getPreStats2(), B, w->L, FP_STATS_PRE2); add_stats(config->getPostStats2(), B, w->L, FP_STATS_POST2); }
    FilterResult* fr = config->getFilterResult();
    const int64_t* F = B + w->L.off_filter;
    for (int i = 0; i < FILTER_RESULT_TYPES; i++) fr->mFilterReadStats[i] += F[FP_FR_READSTATS + i];
    fr->mTrimmedAdapterRead += F[FP_FR_ADAPTER_READS];
    /* mTrimmedAdapterBases: added by FilterResult::addAdapterTrimmed when the events are replayed */
    for (int b = 0; b < 4; b++) { fr->mTrimmedPolyXReads[b] += F[FP_FR_POLYX_READS + b]; fr->mTrimmedPolyXBases[b] += F[FP_FR_POLYX_BASES + b]; }
    for (int i = 0; i < 64; i++) fr->mCorrectionMatrix[i] += F[FP_FR_CORRECTION + i];
    fr->mCorrectedReads += F[FP_FR_CORRECTED_READS];
    fr->mMergedPairs += F[FP_FR_MERGED_PAIRS];                                 /* config->addMergedPairs(mergedCount) :693-695 */
    if (isize) for (int i = 0; i < w->L.isize_bins; i++) if (B[w->L.off_isize + i]) isize[i] += B[w->L.off_isize + i];
    if (fp_counters_reset(w->ctx) != FP_OK) die("fp_counters_reset");
}

/* FilterResult::addAdapterTrimmed calls of the pack, in input order, through the reference's own function (maps, caps, base count) */
void replay_events(GpuWorker* w, uint64_t n_events, const std::vector<int64_t>& unit2pack, FilterResult* fr) {
    if (n_events > w->events.size()) die("adapter event list overflow");
    std::sort(w->events.begin(), w->events.begin() + n_events, [](const fp_adapter_event& a, const fp_adapter_event& b) {
        return a.unit != b.unit ? a.unit < b.unit : a.key < b.key; });
    auto text = [&](const fp_adapter_event& e) -> std::string {
        if (e.kind == FP_EV_ADAPTER) return w->adapters[e.adapter].substr(0, e.len);
        return std::string((const char*)w->seq[e.which] + (size_t)e.unit * w->stride + e.start, e.len);
    };
    (void)unit2pack;
    for (uint64_t i = 0; i < n_events; i++) {
        const fp_adapter_event& e = w->events[i];
        if (e.kind == FP_EV_PAIR) {
            const fp_adapter_event& e2 = w->events[i + 1];
            fr->addAdapterTrimmed(text(e), text(e2));
            i++;
        } else fr->addAdapterTrimmed(text(e), e.which != 0);
    }
}

int g_trace = -1;
void trace(const char* what, long n) {
    if (g_trace < 0) g_trace = getenv("FASTP_B200_TRACE") ? 1 : 0;
    if (g_trace) fprintf(stderr, "[fastp_b200 binding] %s: %ld units on the device\n", what, n);
}
void trace_stock(const char* what, long n) {                                   /* an option set the device path does not cover */
    if (g_trace < 0) g_trace = getenv("FASTP_B200_TRACE") ? 1 : 0;
    if (g_trace) fprintf(stderr, "[fastp_b200 binding] %s: %ld units on the stock body\n", what, n);
}

}  // namespace

/* ------------------------------------------------------------------------------------------------------------------------ */
bool SingleEndProcessor::processSingleEnd(ReadPack* pack, ThreadConfig* config) {
    int maxLen = 0;
    for (int p = 0; p < pack->count; p++) maxLen = std::max(maxLen, pack->data[p]->length());
    GpuWorker* w = supported(mOptions, false) && maxLen <= FP_MAX_STRIDE ? worker_for(this, mOptions, false, config->getThreadId(), maxLen, pack->count) : nullptr;
    if (!w) { trace_stock("processSingleEnd", pack->count); return processSingleEnd_cpu(pack, config); }

    string outstr, failedOut;
    outstr.reserve(pack->count * 320);
    int tid = config->getThreadId();
    int readPassed = 0;
    std::vector<int> kept; kept.reserve(pack->count);
    std::vector<char> dedup(pack->count, 0);
    for (int p = 0; p < pack->count; p++) {                                   /* host-only steps, in the reference's order (:204-230) */
        Read* or1 = pack->data[p];
        if (mDuplicate) { bool isDup = mDuplicate->checkRead(or1); if (mOptions->duplicate.dedup && isDup) dedup[p] = 1; }
        if (mOptions->indexFilter.enabled && mFilter->filterByIndex(or1)) {
            config->getPreStats1()->statRead(or1);                             /* counted before it is dropped (:208) */
            recycleToPool(tid, or1); pack->data[p] = NULL;
            continue;
        }
        if (mOptions->fixMGI) or1->fixMGI();
        stage(w, 0, (int64_t)kept.size(), or1);
        kept.push_back(p);
    }
    const int64_t n = (int64_t)kept.size();
    uint64_t nev = 0;
    if (n > 0) {
        fp_batch b; memset(&b, 0, sizeof(b));
        b.n = n; b.stride = w->stride; b.seq1 = w->seq[0]; b.qual1 = w->qual[0]; b.len1 = w->len[0];
        fp_set_host_event_sink(w->ctx, w->events.data(), w->events.size(), &nev);
        if (fp_process_se_host(w->ctx, &b, w->res[0]) != FP_OK) die("fp_process_se_host");
        replay_events(w, nev, std::vector<int64_t>(), config->getFilterResult());
        add_counters(w, config, false, nullptr);
        trace("processSingleEnd", (long)n);
    }
    for (int64_t i = 0; i < n; i++) {                                          /* the tail of the reference loop (:273-296) */
        const int p = kept[i];
        Read* or1 = pack->data[p];
        Read* r1 = unstage(w, 0, i, or1);
        const int result = w->res[0][i].verdict;
        if (!dedup[p]) {
            if (r1 != NULL && result == PASS_FILTER) { r1->appendToString(&outstr); readPassed++; }
            else if (mFailedWriter) or1->appendToStringWithTag(&failedOut, FAILED_TYPES[result]);
        }
        recycleToPool(tid, or1);
    }
    if (mOptions->split.enabled) { if (!mOptions->out1.empty()) config->getWriter1()->writeString(outstr); }
    if (mLeftWriter) mLeftWriter->input(tid, new string(std::move(outstr)));
    if (mFailedWriter) mFailedWriter->input(tid, new string(std::move(failedOut)));
    if (mOptions->split.byFileLines) config->markProcessed(readPassed); else config->markProcessed(pack->count);
    delete pack->data;
    delete pack;
    mPackProcessedCounter.fetch_add(1, std::memory_order_release);
    mBackpressureCV.notify_all();
    return true;
}

/* ------------------------------------------------------------------------------------------------------------------------ */
bool PairEndProcessor::processPairEnd(ReadPack* leftPack, ReadPack* rightPack, ThreadConfig* config) {
    const int count = std::min(leftPack->count, rightPack->count);
    int maxLen = 0;
    for (int p = 0; p < count; p++) maxLen = std::max(maxLen, std::max(leftPack->data[p]->length(), rightPack->data[p]->length()));
    GpuWorker* w = supported(mOptions, mOverlappedWriter != NULL) && maxLen <= 256 ? worker_for(this, mOptions, true, config->getThreadId(), maxLen, count) : nullptr;
    if (!w) { trace_stock("processPairEnd", count); return processPairEnd_cpu(leftPack, rightPack, config); }

    if (leftPack->count != rightPack->count) {                                 /* :363-370 */
        cerr << endl;
        cerr << "WARNING: different read numbers of the " << mPackProcessedCounter << " pack" << endl;
        cerr << "Read1 pack size: " << leftPack->count << endl;
        cerr << "Read2 pack size: " << rightPack->count << endl;
        cerr << "Ignore the unmatched reads" << endl << endl;
        shouldStopReading = true;
    }
    int tid = config->getThreadId();
    string outstr1, outstr2, unpairedOut1, unpairedOut2;
    string singleOutput, mergedOutput, failedOut, overlappedOut;
    const size_t estimatedCapacity = leftPack->count * 320;
    outstr1.reserve(estimatedCapacity);
    outstr2.reserve(estimatedCapacity);
    int readPassed = 0;

    std::vector<int> kept; kept.reserve(count);
    std::vector<char> dedup(count, 0);
    for (int p = 0; p < count; p++) {                                          /* host-only steps, in the reference's order (:383-420) */
        Read* or1 = leftPack->data[p];
        Read* or2 = rightPack->data[p];
        if (mDuplicate) { bool isDup = mDuplicate->checkPair(or1, or2); if (mOptions->duplicate.dedup && isDup) dedup[p] = 1; }
        if (mOptions->indexFilter.enabled && mFilter->filterByIndex(or1, or2)) {
            config->getPreStats1()->statRead(or1);                             /* counted before they are dropped (:393-394) */
            config->getPreStats2()->statRead(or2);
            recycleToPool1(tid, or1); leftPack->data[p] = NULL;
            recycleToPool2(tid, or2); rightPack->data[p] = NULL;
            continue;
        }
        if (mOptions->fixMGI) { or1->fixMGI(); or2->fixMGI(); }
        stage(w, 0, (int64_t)kept.size(), or1);
        stage(w, 1, (int64_t)kept.size(), or2);
        kept.push_back(p);
    }
    const int64_t n = (int64_t)kept.size();
    uint64_t nev = 0, npatch = 0;
    if (n > 0) {
        fp_batch b; memset(&b, 0, sizeof(b));
        b.n = n; b.stride = w->stride;
        b.seq1 = w->seq[0]; b.qual1 = w->qual[0]; b.len1 = w->len[0]; b.seq2 = w->seq[1]; b.qual2 = w->qual[1]; b.len2 = w->len[1];
        fp_set_host_event_sink(w->ctx, w->events.data(), w->events.size(), &nev);
        if (fp_process_pe_host_patches(w->ctx, &b, w->res[0], w->res[1], w->ov, w->patches.data(), w->patches.size(), &npatch) != FP_OK) die("fp_process_pe_host");
        replay_events(w, nev, std::vector<int64_t>(), config->getFilterResult());
        add_counters(w, config, true, mInsertSizeHist);
        trace("processPairEnd", (long)n);
    }
    for (int64_t i = 0; i < n; i++) {                                          /* the tail of the reference loop (:563-642) */
        const int p = kept[i];
        Read* or1 = leftPack->data[p];
        Read* or2 = rightPack->data[p];
        Read* r1 = unstage(w, 0, i, or1);
        Read* r2 = unstage(w, 1, i, or2);
        if (r1 == NULL || r2 == NULL) {
            /* the reference stops working on a pair as soon as one read is dropped (every later step is guarded by r1 && r2), but the
               other read keeps what trimAndCut did to it: the device reports exactly that window */
        }
        const int result1 = w->res[0][i].verdict, result2 = w->res[1][i].verdict;
        bool mergeProcessed = false;
        if (mOptions->merge.enabled && r1 && r2) {                             /* merging mode :519-560 */
            if (w->res[0][i].flags & FP_F_MERGED) {
                if (result1 == PASS_FILTER) {
                    OverlapResult ov;
                    ov.overlapped = true; ov.hasGap = false;
                    ov.offset = w->ov[i].offset; ov.overlap_len = w->ov[i].overlap_len; ov.diff = w->ov[i].diff;
                    Read* merged = OverlapAnalysis::merge(r1, r2, ov);         /* the reference's own string work (names included) */
                    merged->appendToString(&mergedOutput);
                    readPassed++;
                    recycleToPool1(tid, merged);
                }
                mergeProcessed = true;
            } else if (mOptions->merge.includeUnmerged) {
                if (result1 == PASS_FILTER && !dedup[p]) r1->appendToString(&mergedOutput);
                if (result2 == PASS_FILTER && !dedup[p]) r2->appendToString(&mergedOutput);
                if (result1 == PASS_FILTER && result2 == PASS_FILTER) readPassed++;
                mergeProcessed = true;
            }
        }
        if (!mergeProcessed && !dedup[p]) {
            if (r1 != NULL && result1 == PASS_FILTER && r2 != NULL && result2 == PASS_FILTER) {
                if (mOptions->outputToSTDOUT && !mOptions->merge.enabled) { r1->appendToString(&singleOutput); r2->appendToString(&singleOutput); }
                else { r1->appendToString(&outstr1); r2->appendToString(&outstr2); }
                readPassed++;
            } else if (r1 != NULL && result1 == PASS_FILTER) {
                if (mUnpairedLeftWriter) {
                    r1->appendToString(&unpairedOut1);
                    if (mFailedWriter) or2->appendToStringWithTag(&failedOut, FAILED_TYPES[result2]);
                } else if (mFailedWriter) {
                    or1->appendToStringWithTag(&failedOut, "paired_read_is_failing");
                    or2->appendToStringWithTag(&failedOut, FAILED_TYPES[result2]);
                }
            } else if (r2 != NULL && result2 == PASS_FILTER) {
                if (mUnpairedRightWriter) {
                    r2->appendToString(&unpairedOut2);
                    if (mFailedWriter) or1->appendToStringWithTag(&failedOut, FAILED_TYPES[result1]);
                } else if (mUnpairedLeftWriter) {
                    r2->appendToString(&unpairedOut1);
                    if (mFailedWriter) or1->appendToStringWithTag(&failedOut, FAILED_TYPES[result1]);
                } else if (mFailedWriter) {
                    or1->appendToStringWithTag(&failedOut, FAILED_TYPES[result1]);
                    or2->appendToStringWithTag(&failedOut, "paired_read_is_failing");
                }
            }
        }
        recycleToPool1(tid, or1);
        recycleToPool2(tid, or2);
    }
    for (int p = count; p < leftPack->count; p++) if (leftPack->data[p]) recycleToPool1(tid, leftPack->data[p]);
    for (int p = count; p < rightPack->count; p++) if (rightPack->data[p]) recycleToPool2(tid, rightPack->data[p]);

    if (mOptions->split.enabled) {
        if (!mOptions->out1.empty()) config->getWriter1()->writeString(outstr1);
        if (!mOptions->out2.empty()) config->getWriter2()->writeString(outstr2);
    }
    if (mMergedWriter) mMergedWriter->input(tid, new string(std::move(mergedOutput)));
    if (mFailedWriter) mFailedWriter->input(tid, new string(std::move(failedOut)));
    if (mOverlappedWriter) mOverlappedWriter->input(tid, new string(std::move(overlappedOut)));
    if (mRightWriter && mLeftWriter) {
        mLeftWriter->input(tid, new string(std::move(outstr1)));
        mRightWriter->input(tid, new string(std::move(outstr2)));
    } else if (mLeftWriter) {
        if (mOptions->merge.enabled && mOptions->outputToSTDOUT) mLeftWriter->input(tid, new string(std::move(mergedOutput)));   /* :672-675 */
        else mLeftWriter->input(tid, new string(std::move(singleOutput)));
    }
    if (mUnpairedLeftWriter && mUnpairedRightWriter) {
        mUnpairedLeftWriter->input(tid, new string(std::move(unpairedOut1)));
        mUnpairedRightWriter->input(tid, new string(std::move(unpairedOut2)));
    } else if (mUnpairedLeftWriter) {
        mUnpairedLeftWriter->input(tid, new string(std::move(unpairedOut1)));
    }
    if (mOptions->split.byFileLines) config->markProcessed(readPassed); else config->markProcessed(leftPack->count);
    delete[] leftPack->data;
    delete[] rightPack->data;
    delete leftPack;
    delete rightPack;
    mPackProcessedCounter.fetch_add(1, std::memory_order_release);
    mBackpressureCV.notify_all();
    return true;
}
