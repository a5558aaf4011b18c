/*
 * gpu_worker.cpp -- the host shim that replaces "N CPU workers" by "stage -> GPU -> unstage"
 * (SURVEY.md App. E.4).  stage() copies Read::mSeq / mQuality bytes into pinned fixed-stride SoA rows
 * (names / strands stay in the Read objects); the C-ABI call runs the whole operator chain on the device;
 * unstage() applies each fp_read_result exactly as the reference's in-place string edits would
 * (erase(0,front); resize(len); corrected bytes copied back) and the unchanged tail of the reference loop
 * (output string building src/peprocessor.cpp:575-620) runs here on the verdicts.
 */
#include "fastp_host.h"
#include <cstdio>
#include <cstring>
#include <algorithm>

namespace fastp_b200 {

void Options::toParams(fp_params* p, std::vector<const char*>& fastaKeep, std::vector<const char*>& ovr1Keep, std::vector<const char*>& ovr2Keep) const {
    fp_params_default(p, paired ? 1 : 0);
    p->trim_front1 = trim.front1; p->trim_tail1 = trim.tail1; p->trim_front2 = trim.front2; p->trim_tail2 = trim.tail2;
    p->max_len1 = trim.maxLen1; p->max_len2 = trim.maxLen2;
    p->cut_front = qualityCut.enabledFront; p->cut_tail = qualityCut.enabledTail; p->cut_right = qualityCut.enabledRight;
    p->cut_front_window = qualityCut.windowSizeFront; p->cut_front_quality = qualityCut.qualityFront;
    p->cut_tail_window = qualityCut.windowSizeTail; p->cut_tail_quality = qualityCut.qualityTail;
    p->cut_right_window = qualityCut.windowSizeRight; p->cut_right_quality = qualityCut.qualityRight;
    p->polyg_enabled = polyGTrim.enabled; p->polyg_min_len = polyGTrim.minLen;
    p->polyx_enabled = polyXTrim.enabled; p->polyx_min_len = polyXTrim.minLen;
    p->adapter_enabled = adapter.enabled; p->has_seq_r1 = adapter.hasSeqR1; p->has_seq_r2 = adapter.hasSeqR2;
    p->adapter_seq_r1 = adapter.sequence.c_str(); p->adapter_seq_r2 = adapter.sequenceR2.c_str();
    fastaKeep.clear();
    if (adapter.hasFasta) for (auto& s : adapter.seqsInFasta) fastaKeep.push_back(s.c_str());
    p->n_fasta_adapters = (int)fastaKeep.size(); p->fasta_adapters = fastaKeep.empty() ? nullptr : fastaKeep.data();
    p->allow_gap_overlap_trimming = adapter.allowGapOverlapTrimming; p->dimer_max_len = adapter.dimerMaxLen;
    p->correction_enabled = correction.enabled || merge.enabled;           /* options.cpp:120-121 */
    p->merge_enabled = merge.enabled; p->merge_include_unmerged = merge.includeUnmerged;
    p->overlap_require = overlapRequire; p->overlap_diff_limit = overlapDiffLimit; p->overlap_diff_percent_limit = overlapDiffPercentLimit;
    p->qual_filter_enabled = qualfilter.enabled; p->qualified_qual = (unsigned char)qualfilter.qualifiedQual;
    p->unqualified_percent_limit = qualfilter.unqualifiedPercentLimit; p->n_base_limit = qualfilter.nBaseLimit; p->avg_qual_req = qualfilter.avgQualReq;
    p->length_filter_enabled = lengthFilter.enabled; p->length_required = lengthFilter.requiredLength; p->length_limit = lengthFilter.maxLength;
    p->complexity_filter_enabled = complexityFilter.enabled; p->complexity_threshold = complexityFilter.threshold;
    p->insert_size_max = insertSizeMax; p->seq_len1 = seqLen1; p->seq_len2 = seqLen2;
    p->overrep_enabled = overRepAnalysis.enabled; p->overrep_sampling = overRepAnalysis.sampling;
    ovr1Keep.clear(); ovr2Keep.clear();
    for (auto& kv : overRepSeqs1) ovr1Keep.push_back(kv.first.c_str());
    for (auto& kv : overRepSeqs2) ovr2Keep.push_back(kv.first.c_str());
    p->n_overrep1 = (int)ovr1Keep.size(); p->overrep_seqs1 = ovr1Keep.empty() ? nullptr : ovr1Keep.data();
    p->n_overrep2 = (int)ovr2Keep.size(); p->overrep_seqs2 = ovr2Keep.empty() ? nullptr : ovr2Keep.data();
}

void FilterResult::fill(const int64_t* B, const fp_counter_layout& L) {
    const int64_t* F = B + L.off_filter;
    for (int i = 0; i < FP_FILTER_RESULT_TYPES; i++) mFilterReadStats[i] = F[FP_FR_READSTATS + i];
    mTrimmedAdapterRead = F[FP_FR_ADAPTER_READS]; mTrimmedAdapterBases = F[FP_FR_ADAPTER_BASES];
    for (int b = 0; b < 4; b++) { mTrimmedPolyXReads[b] = F[FP_FR_POLYX_READS + b]; mTrimmedPolyXBases[b] = F[FP_FR_POLYX_BASES + b]; }
    for (int i = 0; i < 64; i++) mCorrectionMatrix[i] = F[FP_FR_CORRECTION + i];
    mCorrectedReads = F[FP_FR_CORRECTED_READS]; mMergedPairs = F[FP_FR_MERGED_PAIRS];
}

void Stats::fillOverRep(const int64_t* B, const fp_counter_layout& L, int which, const std::vector<const char*>& keys) {
    const int side = which >> 1;
    for (int k = 0; k < L.n_overrep[side] && k < (int)keys.size(); k++) {
        mOverRepSeq[keys[k]] = B[fp_off_overrep_count(&L, which, k)];
        std::vector<long>& d = mOverRepSeqDist[keys[k]];
        d.assign(L.overrep_len[side], 0);
        for (int q = 0; q < L.overrep_len[side]; q++) d[q] = B[fp_off_overrep_dist(&L, which, k, q)];
    }
}

void Stats::fill(const int64_t* B, const fp_counter_layout& L, int which) {
    mBufLen = L.cycles;
    for (int b = 0; b < 8; b++) {
        mCycleQ30Bases[b].assign(L.cycles, 0); mCycleQ20Bases[b].assign(L.cycles, 0);
        mCycleBaseContents[b].assign(L.cycles, 0); mCycleBaseQual[b].assign(L.cycles, 0);
        for (int c = 0; c < L.cycles; c++) {
            mCycleQ30Bases[b][c] = B[fp_off_cycle(&L, which, 0 * 8 + b, c)];
            mCycleQ20Bases[b][c] = B[fp_off_cycle(&L, which, 1 * 8 + b, c)];
            mCycleBaseContents[b][c] = B[fp_off_cycle(&L, which, 2 * 8 + b, c)];
            mCycleBaseQual[b][c] = B[fp_off_cycle(&L, which, 3 * 8 + b, c)];
        }
    }
    mCycleTotalBase.assign(L.cycles, 0); mCycleTotalQual.assign(L.cycles, 0);
    for (int c = 0; c < L.cycles; c++) { mCycleTotalBase[c] = B[fp_off_cycle(&L, which, 32, c)]; mCycleTotalQual[c] = B[fp_off_cycle(&L, which, 33, c)]; }
    mKmer.assign(FP_KMER_BINS, 0);
    for (int k = 0; k < FP_KMER_BINS; k++) mKmer[k] = B[fp_off_kmer(&L, which, k)];
    for (int q = 0; q < FP_QUAL_BINS; q++) mBaseQualHistogram[q] = B[fp_off_qualhist(&L, which, q)];
    mReads = B[fp_off_reads(&L, which)]; mLengthSum = B[fp_off_length_sum(&L, which)];
    /* Stats::summarize src/stats.cpp:102-182 */
    mCycles = L.cycles; mBases = 0;
    for (int c = 0; c < L.cycles; c++) { mBases += mCycleTotalBase[c]; if (mCycleTotalBase[c] == 0) { mCycles = c; break; } }
    mQ20Total = mQ30Total = 0;
    for (int b = 0; b < 8; b++) for (int c = 0; c < mCycles; c++) { mQ20Total += mCycleQ20Bases[b][c]; mQ30Total += mCycleQ30Bases[b][c]; }
}

GpuChainWorker::GpuChainWorker(const Options* opt, int maxReadLen, int device, int64_t maxBatch) : mOptions(opt) {
    opt->toParams(&mParams, mFastaKeep, mOvr1Keep, mOvr2Keep);
    mStride = std::max(16, (maxReadLen + 15) / 16 * 16);
    mCap = maxBatch;
    /* a merged read is up to two rows long: the per-cycle counters need that many cycles */
    int rc = fp_ctx_create(&mParams, device, maxBatch, mStride, mParams.merge_enabled ? 2 * mStride : mStride, &mCtx);
    if (rc != FP_OK) { mError = fp_last_error(); mCtx = nullptr; return; }
    const int sides = opt->paired ? 2 : 1;
    for (int s = 0; s < sides; s++) {
        rc |= fp_host_alloc((void**)&mSeq[s], (size_t)mCap * mStride);
        rc |= fp_host_alloc((void**)&mQual[s], (size_t)mCap * mStride);
        rc |= fp_host_alloc((void**)&mLen[s], (size_t)mCap * 2);
        rc |= fp_host_alloc((void**)&mRes[s], (size_t)mCap * sizeof(fp_read_result));
    }
    if (opt->paired) rc |= fp_host_alloc((void**)&mOv, (size_t)mCap * sizeof(fp_ov_result));
    if (rc != FP_OK) { mError = fp_last_error(); fp_ctx_destroy(mCtx); mCtx = nullptr; }
}

GpuChainWorker::~GpuChainWorker() {
    for (int s = 0; s < 2; s++) { if (mSeq[s]) fp_host_free(mSeq[s]); if (mQual[s]) fp_host_free(mQual[s]); if (mLen[s]) fp_host_free(mLen[s]); if (mRes[s]) fp_host_free(mRes[s]); }
    if (mOv) fp_host_free(mOv);
    if (mCtx) fp_ctx_destroy(mCtx);
}

bool GpuChainWorker::stage(ReadPack* pack, int side, int64_t n) {
    for (int64_t i = 0; i < n; i++) {
        Read* r = pack->data[i];
        const int len = r->length();
        if (len > mStride) { mError = "read longer than the staging stride"; return false; }
        uint8_t* s = mSeq[side] + i * mStride; uint8_t* q = mQual[side] + i * mStride;
        memcpy(s, r->mSeq->data(), len); memcpy(q, r->mQuality->data(), len);
        mLen[side][i] = (uint16_t)len;
    }
    return true;
}

void GpuChainWorker::unstage(Read* r, const fp_read_result& res, const uint8_t* seqRow, const uint8_t* qualRow, bool corrected) {
    if (res.flags & FP_F_DROPPED) return;                     /* r == NULL in the reference */
    if (corrected) { r->mSeq->assign((const char*)seqRow, r->mSeq->size()); r->mQuality->assign((const char*)qualRow, r->mQuality->size()); }
    if (res.front) { r->mSeq->erase(0, res.front); r->mQuality->erase(0, res.front); }      /* filter.cpp:199-202 */
    r->mSeq->resize(res.len); r->mQuality->resize(res.len);
}

bool GpuChainWorker::processSingleEnd(ReadPack* pack, std::string* outstr, std::string* failedOut) {
    const int64_t n = pack->count;
    if (mCtx && n <= mCap && stage(pack, 0, n)) {
        fp_batch b; memset(&b, 0, sizeof(b));
        b.n = n; b.stride = mStride; b.seq1 = mSeq[0]; b.qual1 = mQual[0]; b.len1 = mLen[0];
        if (fp_process_se_host(mCtx, &b, mRes[0]) != FP_OK) mError = fp_last_error();
        else for (int64_t i = 0; i < n; i++) {
            Read* r = pack->data[i];
            const fp_read_result& res = mRes[0][i];
            unstage(r, res, mSeq[0] + i * mStride, mQual[0] + i * mStride, false);
            if (!(res.flags & FP_F_DROPPED) && res.verdict == FP_PASS_FILTER) r->appendToString(outstr);   /* seprocessor.cpp:281-286 */
            else if (failedOut) r->appendToString(failedOut);
        }
    } else if (mError.empty()) mError = "pack larger than maxBatch";
    for (int i = 0; i < pack->count; i++) delete pack->data[i];      /* ownership: seprocessor.cpp:288-320 */
    delete[] pack->data; delete pack;
    return true;
}

bool GpuChainWorker::processPairEnd(ReadPack* leftPack, ReadPack* rightPack, std::string* outstr1, std::string* outstr2, std::string* failedOut) {
    const int64_t n = std::min(leftPack->count, rightPack->count);    /* peprocessor.cpp:363-370,383 */
    if (mCtx && n <= mCap && stage(leftPack, 0, n) && stage(rightPack, 1, n)) {
        fp_batch b; memset(&b, 0, sizeof(b));
        b.n = n; b.stride = mStride; b.seq1 = mSeq[0]; b.qual1 = mQual[0]; b.len1 = mLen[0]; b.seq2 = mSeq[1]; b.qual2 = mQual[1]; b.len2 = mLen[1];
        if (fp_process_pe_host(mCtx, &b, mRes[0], mRes[1], mOv) != FP_OK) mError = fp_last_error();
        else for (int64_t i = 0; i < n; i++) {
            Read *r1 = leftPack->data[i], *r2 = rightPack->data[i];
            const fp_read_result &a = mRes[0][i], &c = mRes[1][i];
            unstage(r1, a, mSeq[0] + i * mStride, mQual[0] + i * mStride, a.flags & FP_F_CORRECTED);
            unstage(r2, c, mSeq[1] + i * mStride, mQual[1] + i * mStride, c.flags & FP_F_CORRECTED);
            const bool p1 = !(a.flags & FP_F_DROPPED) && a.verdict == FP_PASS_FILTER, p2 = !(c.flags & FP_F_DROPPED) && c.verdict == FP_PASS_FILTER;
            if (p1 && p2) { r1->appendToString(outstr1); r2->appendToString(outstr2); }      /* peprocessor.cpp:577-593 */
            else if (failedOut) { r1->appendToString(failedOut); r2->appendToString(failedOut); }
        }
    } else if (mError.empty()) mError = "pack larger than maxBatch";
    for (int i = 0; i < leftPack->count; i++) delete leftPack->data[i];       /* ownership: peprocessor.cpp:624-702 */
    for (int i = 0; i < rightPack->count; i++) delete rightPack->data[i];
    delete[] leftPack->data; delete[] rightPack->data; delete leftPack; delete rightPack;
    return true;
}

bool GpuChainWorker::processFastqText(const char* text1, size_t n1, const char* text2, size_t n2, bool final, bool phred64,
                                      std::string* const outs[FQ_TEXT_OUTS], size_t* consumed1, size_t* consumed2, long* units) {
    const bool paired = mParams.paired != 0, merging = paired && mParams.merge_enabled;
    const bool ilIn = paired && mIlIn, ilOut = paired && mIlOut;
    if (ilIn) n2 = 0;                                           /* both mates are in text1 */
    int64_t nu = 0, c1 = 0, c2 = 0;
    fp_fastq_info i1, i2;
    const uint8_t* t1 = reinterpret_cast<const uint8_t*>(text1); const uint8_t* t2 = paired && !ilIn ? reinterpret_cast<const uint8_t*>(text2) : nullptr;
    const size_t both = n1 + (paired ? n2 : 0);
    const size_t side2 = ilIn ? n1 : n2;                        /* the text that holds read 2 */
    /* what each stream can hold at most: a side's reads (both sides' when interleaved); on the merged stream everything both inputs hold, each
       merged read with its name suffix (one per pair, i.e. per 8 lines at least); on unpaired1 reads of either side; on the failed stream
       reads of either side, each with a tag of up to 24 bytes (a record takes 6 bytes at least); on --overlapped_out at most one record of
       read 1 per pair, never longer than read 1's input record */
    std::string* want[FQ_TEXT_OUTS] = {merging ? outs[FP_FQ_OUT_MERGED] : nullptr, outs[FP_FQ_OUT_R1], paired && !ilOut ? outs[FP_FQ_OUT_R2] : nullptr,
                                       paired ? outs[FP_FQ_OUT_UNPAIRED1] : nullptr, paired ? outs[FP_FQ_OUT_UNPAIRED2] : nullptr, outs[FP_FQ_OUT_FAILED],
                                       paired ? outs[FQ_OUT_OVERLAPPED] : nullptr};
    const size_t cap[FQ_TEXT_OUTS] = {n1 + n2 + (n1 / 8 + 1) * 40 + 64, (ilOut ? both : n1) + 64, side2 + 64, both + 64, side2 + 64,
                                      both + (both / 6 + 2) * 24 + 64, n1 + 64};
    uint8_t* bufs[FQ_TEXT_OUTS]; int64_t caps[FQ_TEXT_OUTS], ob[FQ_TEXT_OUTS] = {0};
    for (int s = 0; s < FQ_TEXT_OUTS; s++) {
        if (want[s]) mTextOut[s].resize(cap[s]);
        bufs[s] = want[s] ? mTextOut[s].data() : nullptr;
        caps[s] = want[s] ? (int64_t)cap[s] : 0;
    }
    /* --overlapped_out is not one of the C-ABI's FP_FQ_OUTS streams: its buffer is attached to the ctx for this call */
    const bool ov = want[FQ_OUT_OVERLAPPED] != nullptr;
    if (ov && fp_fastq_set_overlapped_out(mCtx, bufs[FQ_OUT_OVERLAPPED], caps[FQ_OUT_OVERLAPPED], &ob[FQ_OUT_OVERLAPPED]) != FP_OK) { mError = fp_last_error(); return false; }
    const int rc = fp_fastq_process_host_outs(mCtx, t1, (int64_t)n1, t2, paired ? (int64_t)n2 : 0, final ? 1 : 0, phred64 ? 1 : 0, bufs, caps, ob,
                                              &nu, &c1, paired ? &c2 : nullptr, &i1, paired ? &i2 : nullptr);
    if (ov) fp_fastq_set_overlapped_out(mCtx, nullptr, 0, nullptr);
    if (rc != FP_OK) { mError = fp_last_error(); return false; }
    if (i1.error == FP_FQ_ERR_STRIDE || (paired && i2.error == FP_FQ_ERR_STRIDE)) { mError = "a read is longer than the row stride (raise --max_read_len)"; return false; }
    if (i1.error != FP_FQ_OK || (paired && i2.error != FP_FQ_OK)) {
        const fp_fastq_info& bad = i1.error != FP_FQ_OK ? i1 : i2;
        fprintf(stderr, "%s (record %lld of read%d)\nYour FASTQ may be invalid, please check the tail of your FASTQ file\n",
                bad.error == FP_FQ_ERR_STRAND ? "Expected '+'" : "ERROR: sequence and quality have different length:", (long long)bad.error_record, i1.error != FP_FQ_OK ? 1 : 2);
        mInputEnded = true;
    }
    for (int s = 0; s < FQ_TEXT_OUTS; s++)
        if (want[s]) want[s]->append(reinterpret_cast<const char*>(mTextOut[s].data()), (size_t)ob[s]);
    if (consumed1) *consumed1 = (size_t)c1;
    if (consumed2) *consumed2 = (size_t)c2;
    if (units) *units = (long)nu;
    return true;
}

bool GpuChainWorker::finish(Stats* pre1, Stats* post1, Stats* pre2, Stats* post2, FilterResult* fr, std::vector<long>* isize) {
    if (!mCtx) return false;
    fp_counter_layout L;
    fp_ctx_layout(mCtx, &L);
    std::vector<int64_t> B(L.total);
    if (fp_counters_fetch(mCtx, B.data()) != FP_OK) { mError = fp_last_error(); return false; }
    if (pre1) { pre1->fill(B.data(), L, FP_STATS_PRE1); pre1->fillOverRep(B.data(), L, FP_STATS_PRE1, mOvr1Keep); }
    if (post1) { post1->fill(B.data(), L, FP_STATS_POST1); post1->fillOverRep(B.data(), L, FP_STATS_POST1, mOvr1Keep); }
    if (L.n_stats == 4) {
        if (pre2) { pre2->fill(B.data(), L, FP_STATS_PRE2); pre2->fillOverRep(B.data(), L, FP_STATS_PRE2, mOvr2Keep); }
        if (post2) { post2->fill(B.data(), L, FP_STATS_POST2); post2->fillOverRep(B.data(), L, FP_STATS_POST2, mOvr2Keep); }
    }
    if (fr) fr->fill(B.data(), L);
    if (isize) { isize->assign(L.isize_bins, 0); for (int i = 0; i < L.isize_bins; i++) (*isize)[i] = B[L.off_isize + i]; }
    return true;
}

}  // namespace fastp_b200
