/*
 * fastp_host.h -- host side above the C-ABI, in the reference's language (C++), mirroring the reference's
 * data model for the hot path so the shim reads like the code it replaces:
 *   Read / ReadPack          src/read.h:14-47,66-69
 *   Options (hot-path part)  src/options.h (same nested struct and field names)
 *   FilterResult counters    src/filterresult.h:66-79
 *   Stats accumulators       src/stats.h:77-101
 *   GpuChainWorker::processSingleEnd / processPairEnd
 *                            drop-in bodies for SingleEndProcessor::processSingleEnd (src/seprocessor.cpp:197-325)
 *                            and PairEndProcessor::processPairEnd (src/peprocessor.cpp:362-708)
 * No CUDA types here: everything goes through include/fastp_b200.h.
 */
#ifndef FASTP_HOST_H
#define FASTP_HOST_H
#include <map>
#include <string>
#include <vector>
#include <cstdint>
#include "fastp_b200.h"

namespace fastp_b200 {

class Read {                         /* src/read.h:14-47 */
public:
    Read(std::string* name, std::string* seq, std::string* strand, std::string* quality)
        : mName(name), mSeq(seq), mStrand(strand), mQuality(quality) {}
    ~Read() { delete mName; delete mSeq; delete mStrand; delete mQuality; }
    int length() const { return (int)mSeq->length(); }
    void resize(int len) { if (len > length() || len < 0) return; mSeq->resize(len); mQuality->resize(len); }   /* read.cpp:62-67 */
    void appendToString(std::string* target) const {                 /* read.cpp:119-134 */
        target->append(*mName); target->push_back('\n'); target->append(*mSeq); target->push_back('\n');
        target->append(*mStrand); target->push_back('\n'); target->append(*mQuality); target->push_back('\n');
    }
    std::string *mName, *mSeq, *mStrand, *mQuality;
};

struct ReadPack { Read** data; int count; };      /* src/read.h:66-69 */

/* the text path's output streams: FP_FQ_OUT_* (merged, out1, out2, unpaired1, unpaired2, failed), then --overlapped_out */
constexpr int FQ_OUT_OVERLAPPED = FP_FQ_OUTS, FQ_TEXT_OUTS = FP_FQ_OUTS + 1;

/* Same nested names as src/options.h for every field the chain reads. */
struct Options {
    struct { int front1 = 0, tail1 = 0, front2 = 0, tail2 = 0, maxLen1 = 0, maxLen2 = 0; } trim;
    struct { bool enabledFront = false, enabledTail = false, enabledRight = false;
             int windowSizeFront = 4, qualityFront = 20, windowSizeTail = 4, qualityTail = 20, windowSizeRight = 4, qualityRight = 20; } qualityCut;
    struct { bool enabled = false; int minLen = 10; } polyGTrim, polyXTrim;
    struct { bool enabled = true; std::string sequence, sequenceR2; std::vector<std::string> seqsInFasta;
             bool hasSeqR1 = false, hasSeqR2 = false, hasFasta = false, allowGapOverlapTrimming = false; int dimerMaxLen = 2; } adapter;
    struct { bool enabled = false; } correction;
    struct { bool enabled = false, includeUnmerged = false; } merge;              /* options.h:104-121 (text path only) */
    struct { bool enabled = true; char qualifiedQual = '0'; int unqualifiedPercentLimit = 40, nBaseLimit = 5, avgQualReq = 0; } qualfilter;
    struct { bool enabled = true; int requiredLength = 15, maxLength = 0; } lengthFilter;
    struct { bool enabled = false; double threshold = 0.3; } complexityFilter;
    struct { bool enabled = false; int sampling = 20; } overRepAnalysis;           /* options.h:71-80 */
    struct { bool enabled = false; std::vector<std::string> blacklist1, blacklist2; int threshold = 0; } indexFilter;   /* text path only */
    std::map<std::string, long> overRepSeqs1, overRepSeqs2;                        /* options.h:364-365, filled by the Evaluator pre-scan */
    int insertSizeMax = 512, overlapRequire = 30, overlapDiffLimit = 5, overlapDiffPercentLimit = 20;
    int seqLen1 = 151, seqLen2 = 151;
    bool paired = false;
    void toParams(fp_params* p, std::vector<const char*>& fastaKeep, std::vector<const char*>& ovr1Keep, std::vector<const char*>& ovr2Keep) const;
};

/* Merged counters, filled from the device block (fp_counters_fetch). */
struct FilterResult {                 /* src/filterresult.h:66-79 */
    long mFilterReadStats[FP_FILTER_RESULT_TYPES] = {0};
    long mTrimmedAdapterRead = 0, mTrimmedAdapterBases = 0;
    long mTrimmedPolyXReads[4] = {0}, mTrimmedPolyXBases[4] = {0};
    long mCorrectionMatrix[64] = {0};
    long mCorrectedReads = 0, mMergedPairs = 0;
    void fill(const int64_t* block, const fp_counter_layout& L);       /* FilterResult::merge of the device block (filterresult.cpp:38-89) */
};
struct Stats {                        /* src/stats.h:77-101, summarize() src/stats.cpp:102-182 */
    int mCycles = 0, mBufLen = 0;
    long mReads = 0, mBases = 0, mQ20Total = 0, mQ30Total = 0, mLengthSum = 0;
    std::vector<long> mCycleQ30Bases[8], mCycleQ20Bases[8], mCycleBaseContents[8], mCycleBaseQual[8], mCycleTotalBase, mCycleTotalQual;
    std::vector<long> mKmer;          /* 1024 used bins */
    long mBaseQualHistogram[128] = {0};
    std::map<std::string, long> mOverRepSeq;                     /* stats.h:91 */
    std::map<std::string, std::vector<long>> mOverRepSeqDist;    /* stats.h:92 */
    void fillOverRep(const int64_t* block, const fp_counter_layout& L, int which, const std::vector<const char*>& keys);
    void fill(const int64_t* block, const fp_counter_layout& L, int which);
};

class GpuChainWorker {
public:
    /* maxReadLen: longest read the run can contain (sizes the fixed stride); device: CUDA ordinal */
    GpuChainWorker(const Options* opt, int maxReadLen, int device = 0, int64_t maxBatch = 1 << 18);
    ~GpuChainWorker();
    bool ok() const { return mCtx != nullptr; }
    const std::string& error() const { return mError; }

    /* Drop-in bodies.  Like the reference they own and free the packs and every Read in them; passing reads are
     * appended (trimmed, corrected) to outstr*, in input order; `failedOut` (nullable) receives the others.
     * Always return true (src/seprocessor.cpp:324, src/peprocessor.cpp:707); fatal device errors set error(). */
    bool processSingleEnd(ReadPack* pack, std::string* outstr, std::string* failedOut = nullptr);
    bool processPairEnd(ReadPack* leftPack, ReadPack* rightPack, std::string* outstr1, std::string* outstr2, std::string* failedOut = nullptr);

    /* Text path (device FASTQ codec, SURVEY 8f rank 1): one chunk of plain FASTQ text per side in, the passing reads' text out.
     * Replaces the reader's parse (FastqReader::read), the body above and Read::appendToString in one call; `consumed*` says how many
     * bytes of each chunk were used -- the caller prepends the rest to its next chunk.  `final`: no more input follows.
     * `outs`, indexed by FP_FQ_OUT_* and FQ_OUT_OVERLAPPED, receive the streams' text; a NULL entry is not written.  out1 / out2 get the
     * passing reads.  With Options::merge.enabled the merged entry receives the --merged_out stream (merged reads, and with includeUnmerged
     * the passing reads of pairs that did not merge; src/peprocessor.cpp:519-560) and out1 / out2 only the pairs that took neither branch.
     * The unpaired1 / unpaired2 / failed entries receive --unpaired1 / --unpaired2 / --failed_out (src/seprocessor.cpp:280-290,
     * src/peprocessor.cpp:594-620); NULL means that writer does not exist, which decides where a pair with one failing read goes
     * (fp_fastq_process_host_outs).  The unpaired ones are for paired runs without --include_unmerged.  The FQ_OUT_OVERLAPPED entry
     * receives --overlapped_out (src/peprocessor.cpp:488-495, paired runs; fp_fastq_set_overlapped_out). */
    /* true once a reader rejected a record (strand line not '+', |quality| != |sequence|): like FastqReader::read returning NULL the
     * input ENDS there -- the caller stops feeding chunks (src/fastqreader.cpp:349-364) */
    bool inputEnded() const { return mInputEnded; }
    /* text path: Duplicate::checkRead / checkPair on the device at `accuracyLevel` (src/main.cpp:200-209; 0 = off); dedup: drop duplicates (-D) */
    bool setDedup(int accuracyLevel, bool dedup) { return mCtx && fp_fastq_set_dedup(mCtx, accuracyLevel, dedup ? 1 : 0) == FP_OK; }
    /* text path, paired runs: in = mates alternate in text1 (--interleaved_in; pass text2 NULL, n2 0), out = outstr1 receives read 1 then read 2
     * of every pair (--stdout, src/peprocessor.cpp:579-581; not with merging, whose stdout stream is `merged`) and outstr2 nothing */
    bool setInterleaved(bool in, bool out) {
        if (!mCtx || fp_fastq_set_interleaved(mCtx, in ? 1 : 0, out ? 1 : 0) != FP_OK) return false;
        mIlIn = in; mIlOut = out; return true;
    }
    /* text path: --filter_by_index1 / --filter_by_index2 (src/filter.cpp:209-243) with the lists Options::initIndexFiltering loaded */
    bool setIndexFilter(const std::vector<std::string>& list1, const std::vector<std::string>& list2, int threshold) {
        std::vector<const char*> l1, l2;
        for (const std::string& b : list1) l1.push_back(b.c_str());
        for (const std::string& b : list2) l2.push_back(b.c_str());
        return mCtx && fp_fastq_set_index_filter(mCtx, l1.data(), (int64_t)l1.size(), l2.data(), (int64_t)l2.size(), threshold) == FP_OK;
    }
    bool dupTotals(long* total, long* dups) { int64_t t = 0, d = 0; if (!mCtx || fp_dup_totals(mCtx, &t, &d) != FP_OK) return false; *total = (long)t; *dups = (long)d; return true; }
    bool processFastqText(const char* text1, size_t n1, const char* text2, size_t n2, bool final, bool phred64,
                          std::string* const outs[FQ_TEXT_OUTS], size_t* consumed1, size_t* consumed2, long* units);

    /* end of run: what Stats::merge / FilterResult::merge hand to the reporters (src/peprocessor.cpp:217-234) */
    bool finish(Stats* pre1, Stats* post1, Stats* pre2, Stats* post2, FilterResult* fr, std::vector<long>* insertSizeHist);

private:
    bool stage(ReadPack* pack, int side, int64_t n);
    void unstage(Read* r, const fp_read_result& res, const uint8_t* seqRow, const uint8_t* qualRow, bool corrected);
    const Options* mOptions;
    fp_ctx* mCtx = nullptr;
    fp_params mParams;
    std::vector<const char*> mFastaKeep, mOvr1Keep, mOvr2Keep;
    int mStride = 0;
    int64_t mCap = 0;
    uint8_t *mSeq[2] = {nullptr, nullptr}, *mQual[2] = {nullptr, nullptr};    /* pinned SoA staging */
    uint16_t* mLen[2] = {nullptr, nullptr};
    fp_read_result* mRes[2] = {nullptr, nullptr};
    fp_ov_result* mOv = nullptr;
    std::vector<uint8_t> mTextOut[FQ_TEXT_OUTS];    /* indexed like processFastqText's outs */
    bool mInputEnded = false;
    bool mIlIn = false, mIlOut = false;
    std::string mError;
};

}  // namespace fastp_b200
#endif
